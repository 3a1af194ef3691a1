"""Argument checks of the device-frame entry points (yb_network_predict_device_frames, yb_network_submit_device_frames):
every invalid argument that can be seen without asking the driver about the pointers is rejected before any device work,
so these run without a GPU; and the Python mirror rejects frames of the wrong dtype, rank, shape, strides or format, here
with stub objects that carry a __cuda_array_interface__."""
import ctypes as C
import os

import numpy as np
import pytest

import ybtest_util as util
from device_frames_util import GOLDEN_NV12, nv12_to_rgb

RGB, BGR, PLANAR, NV12 = 0, 1, 2, 3
P = 0x10000          # never dereferenced: every case below is rejected before the pointer query


@pytest.fixture(scope="module")
def net(tmp_path_factory):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", str(tmp_path_factory.mktemp("device_frames_args")))
    return yb.load_network(cfg, wts, batch=2)


def _frame(w=8, h=8, pitch=None, data=P, chroma=None, plane=0):
    from yolo2_light_b200.api import DeviceFrame
    return DeviceFrame(data, chroma, w, h, 3 * w if pitch is None else pitch, plane)


def _call(net, which, frames, nimg, fmt, max_rows=64):
    """The raw C call; frames: a list of DeviceFrame, or None (a null array)."""
    from yolo2_light_b200 import api
    L = api.lib()
    arr = None if frames is None else (api.DeviceFrame * max(len(frames), 1))(*frames)
    if which == "predict":
        ok = bool(L.yb_network_predict_device_frames(net._h, arr, nimg, fmt, 0, None))
    else:
        ok = L.yb_network_submit_device_frames(net._h, arr, nimg, fmt, 0, 0.5, 0.45, 1, 0, max_rows, None) >= 0
    api._check(ok)


CASES = [   # (frames, nimg, format, message)
    ([_frame()], 0, RGB, "nimg 0 outside 1..2"),
    ([_frame()] * 3, 3, RGB, "nimg 3 outside 1..2"),
    (None, 1, RGB, "null frames array"),
    ([_frame()], 1, 4, "unknown frame format 4"),
    ([_frame()], 1, -1, "unknown frame format -1"),
    ([_frame(), _frame(data=None)], 2, RGB, "frame 1 is null"),
    ([_frame(w=8, h=8, pitch=8)], 1, NV12, "frame 0 has a null chroma plane"),
    ([_frame(w=0)], 1, RGB, "frame 0 has size 0x8"),
    ([_frame(h=-2)], 1, BGR, "frame 0 has size 8x-2"),
    ([_frame(w=7, h=8, pitch=8, chroma=P)], 1, NV12, "frame 0 has size 7x8, NV12 needs an even width and height"),
    ([_frame(w=8, h=5, pitch=8, chroma=P)], 1, NV12, "frame 0 has size 8x5, NV12 needs an even width and height"),
    ([_frame(w=8, pitch=23)], 1, RGB, "frame 0 has pitch 23 below its row of 24 bytes"),
    ([_frame(w=8, pitch=23)], 1, BGR, "frame 0 has pitch 23 below its row of 24 bytes"),
    ([_frame(w=8, pitch=7, plane=64)], 1, PLANAR, "frame 0 has pitch 7 below its row of 8 bytes"),
    ([_frame(w=8, pitch=7, chroma=P)], 1, NV12, "frame 0 has pitch 7 below its row of 8 bytes"),
    ([_frame(w=8, h=8, pitch=8, plane=63)], 1, PLANAR, "frame 0 has plane_stride 63 below pitch \\* h = 64"),
    ([_frame(w=8, h=8, pitch=8, plane=-1)], 1, PLANAR, "frame 0 has plane_stride -1 below pitch \\* h = 64"),
    ([_frame(), _frame(w=40000, h=20000)], 2, RGB, "frame 1 addresses more than INT_MAX bytes"),
    ([_frame(w=16, h=20000, pitch=200000, chroma=P)], 1, NV12, "frame 0 addresses more than INT_MAX bytes"),
    ([_frame(w=1000, h=1000, pitch=1000, plane=1 << 30)], 1, PLANAR, "frame 0 addresses more than INT_MAX bytes"),
]


@pytest.mark.parametrize("which", ["predict", "submit"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_device_frame_calls_reject_bad_arguments(net, which, case):
    import yolo2_light_b200 as yb
    frames, nimg, fmt, msg = CASES[case]
    fn = "predict_device_frames" if which == "predict" else "submit_device_frames"
    with pytest.raises(yb.YbError, match=f"{fn}: " + msg.replace("..", r"\.\.")):
        _call(net, which, frames, nimg, fmt)


@pytest.mark.parametrize("max_rows", [0, -1, 16385])
def test_submit_max_rows_out_of_range(net, max_rows):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match=r"max_rows must be in 1\.\.16384"):
        _call(net, "submit", [_frame()], 1, RGB, max_rows=max_rows)


def test_network_without_three_channels_is_rejected(tmp_path):
    import yolo2_light_b200 as yb
    from yolo2_light_b200 import cfgs
    secs = cfgs.slim(cfgs.yolov3_tiny, 2, 64, 64)
    secs[0][1]["channels"] = "1"
    cfg = cfgs.write_cfg(secs, str(tmp_path / "gray.cfg"))
    wts = cfgs.write_weights(secs, str(tmp_path / "gray.weights"), seed=3)
    gray = yb.load_network(cfg, wts, batch=2)
    assert gray.c == 1
    for which, fn in (("predict", "predict_device_frames"), ("submit", "submit_device_frames")):
        with pytest.raises(yb.YbError, match=f"{fn}: device frames have 3 channels, the network's input has 1"):
            _call(gray, which, [_frame()], 1, RGB)


class Stub:
    """An object that looks like a device array to the Python mirror."""

    def __init__(self, shape, strides=None, typestr="|u1", ptr=P):
        self.__cuda_array_interface__ = {"shape": shape, "strides": strides, "typestr": typestr, "data": (ptr, False),
                                         "version": 3}


def test_python_mirror_builds_the_frame_table(net):
    """What the mirror hands to the C call, for each accepted shape."""
    cases = [
        ("rgb", Stub((6, 8, 3), (40, 3, 1)), dict(data=P, chroma=None, w=8, h=6, pitch=40, plane_stride=0)),
        ("bgr", Stub((6, 8, 3)), dict(data=P, chroma=None, w=8, h=6, pitch=24, plane_stride=0)),
        ("planar", Stub((3, 6, 8), (100, 9, 1)), dict(data=P, chroma=None, w=8, h=6, pitch=9, plane_stride=100)),
        ("nv12", Stub((9, 8), (10, 1)), dict(data=P, chroma=P + 60, w=8, h=6, pitch=10, plane_stride=0)),
        ("nv12", (Stub((6, 8), (16, 1)), Stub((3, 8), (16, 1), ptr=P + 4096)),
         dict(data=P, chroma=P + 4096, w=8, h=6, pitch=16, plane_stride=0)),
        # a one-row UV plane reports contiguous strides whatever its pitch: the Y plane's pitch is used
        ("nv12", (Stub((2, 8), (16, 1)), Stub((1, 8), ptr=P + 4096)),
         dict(data=P, chroma=P + 4096, w=8, h=2, pitch=16, plane_stride=0)),
    ]
    for fmt, f, exp in cases:
        keep, arr, F = net._device_frames([f], fmt, "predict_device_frames")
        from yolo2_light_b200.api import FRAME_FORMATS
        assert F == FRAME_FORMATS[fmt] and keep == [f]
        got = {k: getattr(arr[0], k) for k in exp}
        assert got == exp, (fmt, got, exp)


@pytest.mark.parametrize("frames,fmt,msg", [
    ([Stub((8, 8, 3))], "yuv", "unknown format 'yuv', expected one of rgb, bgr, planar, nv12"),
    ([], "rgb", "0 frames, the network takes 1..2"),
    ([Stub((8, 8, 3))] * 3, "rgb", "3 frames, the network takes 1..2"),
    ([np.zeros((8, 8, 3), np.uint8)], "rgb", "frame 0 must expose __cuda_array_interface__"),
    ([Stub((8, 8, 3)), Stub((8, 8, 3), typestr="<f4")], "rgb", "frame 1 must be a uint8 \\[h, w, 3\\]"),
    ([Stub((8, 24))], "rgb", "frame 0 must be a uint8 \\[h, w, 3\\]"),
    ([Stub((8, 8, 4))], "bgr", "frame 0 must be a uint8 \\[h, w, 3\\]"),
    ([Stub((8, 8, 3), (24, 1, 8))], "rgb", "frame 0 must be a uint8 \\[h, w, 3\\] \\(strides \\(pitch, 3, 1\\)\\) array, "
                                           "got shape \\(8, 8, 3\\) strides \\(24, 1, 8\\)"),
    ([Stub((8, 8, 3), (-24, 3, 1))], "rgb", "frame 0 must be a uint8 .* strides \\(-24, 3, 1\\)"),
    ([Stub((8, 8, 3), (1 << 31, 3, 1))], "rgb", "frame 0 must be a uint8 .* strides \\(2147483648, 3, 1\\)"),
    ([Stub((8, 8, 3))], "planar", "frame 0 must be a uint8 \\[3, h, w\\]"),
    ([Stub((4, 8, 8))], "planar", "frame 0 must be a uint8 \\[3, h, w\\]"),
    ([Stub((3, 8, 8), (64, 8, 2))], "planar", "frame 0 must be a uint8 \\[3, h, w\\] \\(strides \\(plane, pitch, 1\\)\\)"),
    ([Stub((8, 8, 3))], "nv12", "frame 0 must be a uint8 \\[3h/2, w\\]"),
    ([Stub((10, 8))], "nv12", "frame 0: an nv12 array has 3h/2 rows, got 10"),
    ([Stub((12, 8), (8, 2))], "nv12", "frame 0 must be a uint8 \\[3h/2, w\\] \\(strides \\(pitch, 1\\)\\)"),
    ([(Stub((8, 8)),)], "nv12", "frame 0: an nv12 pair is \\(Y \\[h, w\\], UV \\[h/2, w\\]\\), got 1 arrays"),
    ([(Stub((8, 8)), Stub((4, 8), (16, 1)))], "nv12", "frame 0: UV plane \\(4, 8\\) with pitch 16 does not match Y plane \\(8, 8\\)"),
    ([(Stub((8, 8)), Stub((8, 8)))], "nv12", "frame 0: UV plane \\(8, 8\\) with pitch 8 does not match"),
    ([(Stub((8, 8)), Stub((4, 6)))], "nv12", "frame 0: UV plane \\(4, 6\\) with pitch 6 does not match"),
    ([(Stub((8, 8), typestr="|i1"), Stub((4, 8)))], "nv12", "frame 0 must be a uint8 Y \\[h, w\\]"),
])
def test_python_mirror_rejects_bad_frames(net, frames, fmt, msg):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match="predict_device_frames: " + msg.replace("..", r"\.\.")):
        net.predict_device_frames(frames, fmt=fmt)
    with pytest.raises(yb.YbError, match="submit_device_frames: " + msg.replace("..", r"\.\.")):
        net.submit_device_frames(frames, 0.5, fmt=fmt)


def test_nv12_restatement_equals_cv2_fixture():
    """The numpy NV12 -> RGB of the tests equals OpenCV's cvtColor, bit for bit, on the committed fixture (and on the live
    cv2 when it is installed)."""
    g = np.load(GOLDEN_NV12)
    n = len([k for k in g.files if k.startswith("nv12_")])
    assert n >= 5
    sizes = set()
    for i in range(n):
        nv = g[f"nv12_{i}"]
        rgb = nv12_to_rgb(nv)
        sizes.add((nv.shape[1], nv.shape[0] // 3 * 2))
        assert np.array_equal(rgb, g[f"rgb_{i}"]), i
        assert np.array_equal(rgb[..., ::-1], g[f"bgr_{i}"]), i
    assert (2, 2) in sizes and max(w for w, _ in sizes) > 4096
    try:
        import cv2
    except ImportError:
        return
    for i in range(n):
        nv = g[f"nv12_{i}"]
        assert np.array_equal(cv2.cvtColor(nv, cv2.COLOR_YUV2RGB_NV12), g[f"rgb_{i}"]), i
        assert np.array_equal(cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12), g[f"bgr_{i}"]), i


def test_nv12_fixture_walks_every_luma_value_with_extreme_chroma():
    g = np.load(GOLDEN_NV12)
    walk = [g[k] for k in g.files if k.startswith("nv12_") and g[k].shape == (15, 256)]
    assert walk
    nv = walk[0]
    assert all(np.array_equal(nv[r], np.arange(256)) for r in range(10))
    uv = {(int(nv[r, 0]), int(nv[r, 1])) for r in range(10, 15)}
    assert {(0, 0), (0, 255), (255, 0), (255, 255)} <= uv
    assert os.path.getsize(GOLDEN_NV12) < 200_000
