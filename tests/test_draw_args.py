"""Argument checks of yb_network_submit_device_frames_draw: everything yb_network_submit_device_frames rejects, and two
frames with the same data pointer, are rejected before any device work, so these run without a GPU.  And
yb_network_selected_detections has no list for a ticket that was never a collected drawing ticket."""
import ctypes as C

import pytest

import ybtest_util as util

RGB, BGR, PLANAR, NV12 = 0, 1, 2, 3
P = 0x10000          # never dereferenced: every case below is rejected before the pointer query


@pytest.fixture(scope="module")
def net(tmp_path_factory):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", str(tmp_path_factory.mktemp("draw_args")))
    return yb.load_network(cfg, wts, batch=3)


def _frame(w=8, h=8, pitch=None, data=P, chroma=None, plane=0):
    from yolo2_light_b200.api import DeviceFrame
    return DeviceFrame(data, chroma, w, h, 3 * w if pitch is None else pitch, plane)


def _call(net, frames, nimg, fmt, max_rows=64):
    from yolo2_light_b200 import api
    L = api.lib()
    arr = None if frames is None else (api.DeviceFrame * max(len(frames), 1))(*frames)
    api._check(L.yb_network_submit_device_frames_draw(net._h, arr, nimg, fmt, 0, 0.5, 0.45, 0, max_rows, None) >= 0)


CASES = [   # (frames, nimg, format, message)
    ([_frame()], 0, RGB, "nimg 0 outside 1..3"),
    ([_frame()] * 4, 4, RGB, "nimg 4 outside 1..3"),
    (None, 1, RGB, "null frames array"),
    ([_frame()], 1, 4, "unknown frame format 4"),
    ([_frame(), _frame(data=None)], 2, RGB, "frame 1 is null"),
    ([_frame(w=8, h=8, pitch=8)], 1, NV12, "frame 0 has a null chroma plane"),
    ([_frame(data=P), _frame(data=P + 4096, w=8, h=8, pitch=8)], 2, NV12, "frame 0 has a null chroma plane"),
    ([_frame(w=0)], 1, RGB, "frame 0 has size 0x8"),
    ([_frame(w=7, h=8, pitch=8, chroma=P)], 1, NV12, "frame 0 has size 7x8, NV12 needs an even width and height"),
    ([_frame(w=8, pitch=23)], 1, BGR, "frame 0 has pitch 23 below its row of 24 bytes"),
    ([_frame(w=8, h=8, pitch=8, plane=63)], 1, PLANAR, "frame 0 has plane_stride 63 below pitch \\* h = 64"),
    ([_frame(), _frame(w=40000, h=20000, data=P + 4096)], 2, RGB, "frame 1 addresses more than INT_MAX bytes"),
    # the drawing call's own check: frames drawn in place must be distinct
    ([_frame(), _frame()], 2, RGB, "frames 0 and 1 share their data pointer"),
    ([_frame(), _frame(data=P + 4096), _frame(w=16, pitch=48)], 3, BGR, "frames 0 and 2 share their data pointer"),
    ([_frame(data=P + 4096), _frame(), _frame(pitch=24, data=P)], 3, RGB, "frames 1 and 2 share their data pointer"),
    ([_frame(w=8, pitch=8, chroma=P + 64), _frame(w=8, pitch=8, chroma=P + 8192)], 2, NV12,
     "frames 0 and 1 share their data pointer"),
    ([_frame(w=8, pitch=8, plane=64)] * 2, 2, PLANAR, "frames 0 and 1 share their data pointer"),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_draw_call_rejects_bad_arguments(net, case):
    import yolo2_light_b200 as yb
    frames, nimg, fmt, msg = CASES[case]
    with pytest.raises(yb.YbError, match="submit_device_frames_draw: " + msg.replace("..", r"\.\.")):
        _call(net, frames, nimg, fmt)


@pytest.mark.parametrize("max_rows", [0, -1, 16385])
def test_draw_call_rejects_max_rows_out_of_range(net, max_rows):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match=r"submit_device_frames_draw: max_rows must be in 1\.\.16384"):
        _call(net, [_frame()], 1, RGB, max_rows=max_rows)


def test_draw_call_rejects_networks_without_three_channels(tmp_path):
    import yolo2_light_b200 as yb
    from yolo2_light_b200 import cfgs
    secs = cfgs.slim(cfgs.yolov3_tiny, 2, 64, 64)
    secs[0][1]["channels"] = "1"
    cfg = cfgs.write_cfg(secs, str(tmp_path / "gray.cfg"))
    wts = cfgs.write_weights(secs, str(tmp_path / "gray.weights"), seed=3)
    gray = yb.load_network(cfg, wts, batch=2)
    with pytest.raises(yb.YbError, match="submit_device_frames_draw: device frames have 3 channels, the network's input has 1"):
        _call(gray, [_frame()], 1, RGB)


def test_python_mirror_checks_frames_with_the_call_name(net):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match=r"submit_device_frames_draw: 4 frames, the network takes 1\.\.3"):
        net.submit_device_frames_draw([object()] * 4, 0.5)
    with pytest.raises(yb.YbError, match="submit_device_frames_draw: frame 0 must expose __cuda_array_interface__"):
        net.submit_device_frames_draw([bytearray(8)], 0.5)


@pytest.mark.parametrize("ticket", [-1, 0, 1, 2, 3, 1 << 30])
def test_no_selected_list_without_a_collected_drawing_ticket(net, ticket):
    from yolo2_light_b200 import api
    dets, counts = C.POINTER(api.Detection)(), C.POINTER(C.c_int)()
    assert api.lib().yb_network_selected_detections(net._h, ticket, C.byref(dets), C.byref(counts)) == -1
    assert not dets and not counts
    assert net.selected_detections(ticket) is None


def test_detection_record_layout():
    import numpy as np
    from yolo2_light_b200 import api
    assert C.sizeof(api.Detection) == api.DETECTION_DTYPE.itemsize == 28
    assert [api.Detection.__dict__[k].offset for k in api.DETECTION_DTYPE.names] == \
        [api.DETECTION_DTYPE.fields[k][1] for k in api.DETECTION_DTYPE.names]
    assert np.dtype(api.DETECTION_DTYPE).names == ("x", "y", "w", "h", "prob", "cls", "row")
