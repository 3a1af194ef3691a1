"""Argument checks of letterboxing (yb_network_set_letterbox): with it on, a frame whose letterbox size has a side below
2 pixels is rejected by every frame call that resizes, before any device work, with the frame's index and letterbox size;
so these run without a GPU.  With it off the same frames pass the checks (they are stretched as before)."""
import ctypes as C

import numpy as np
import pytest

import ybtest_util as util

BUF = np.zeros(640 * 40 * 3 * 2, np.uint8)
P = BUF.ctypes.data
DEV = 0x10000        # a device-frame pointer that is never dereferenced
# (w, h) -> the message: in a 64 x 64 network a 640 x 10 frame letterboxes to 64 x 1 and a 1 x 40 frame to 1 x 64
THIN = {(640, 10): r"frame 1 \(640x10\) letterboxes to 64x1 in the 64x64 network",
        (1, 40): r"frame 1 \(1x40\) letterboxes to 1x64 in the 64x64 network"}
CALLS = ["predict_frames_u8", "submit_frames_u8", "predict_image_u8", "submit_u8", "predict_device_frames",
         "submit_device_frames"]


@pytest.fixture(scope="module")
def net(tmp_path_factory):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", str(tmp_path_factory.mktemp("letterbox_args")))
    return yb.load_network(cfg, wts, batch=2)


def _call(net, which, w, h):
    """The raw C call with two frames, the second (or, for the one-size calls, both) w x h.  Returns (accepted, ticket)."""
    from yolo2_light_b200 import api
    L = api.lib()
    if which.endswith("device_frames"):
        arr = (api.DeviceFrame * 2)(api.DeviceFrame(DEV, None, 8, 8, 24, 0), api.DeviceFrame(DEV, None, w, h, 3 * w, 0))
        if which == "predict_device_frames":
            return bool(L.yb_network_predict_device_frames(net._h, arr, 2, 0, 0, None)), -1
        t = L.yb_network_submit_device_frames(net._h, arr, 2, 0, 0, 0.5, 0.45, 1, 1, 64, None)
        return t >= 0, t
    elif which in ("predict_image_u8", "submit_u8"):
        if which == "predict_image_u8":
            return bool(L.yb_network_predict_image_u8(net._h, C.c_void_p(P), w, h, 0)), -1
        t = L.yb_network_submit_u8(net._h, C.c_void_p(P), w, h, 0, 0.5, 0.45, 1, 1, 64)
        return t >= 0, t
    else:
        fa = (C.c_void_p * 2)(P, P)
        wa, ha = (C.c_int * 2)(8, w), (C.c_int * 2)(8, h)
        if which == "predict_frames_u8":
            return bool(L.yb_network_predict_frames_u8(net._h, fa, wa, ha, 2, 0)), -1
        t = L.yb_network_submit_frames_u8(net._h, fa, wa, ha, 2, 0, 0.5, 0.45, 1, 1, 64)
        return t >= 0, t


@pytest.mark.parametrize("size", list(THIN), ids=[f"{w}x{h}" for w, h in THIN])
@pytest.mark.parametrize("which", CALLS)
def test_thin_frames_rejected_with_letterbox_on(net, which, size):
    import yolo2_light_b200 as yb
    from yolo2_light_b200 import api
    msg = THIN[size]
    if which in ("predict_image_u8", "submit_u8"):
        msg = msg.replace("frame 1", "frame 0")   # every frame of the one-size calls has the size
    net.set_letterbox(True)
    try:
        with pytest.raises(yb.YbError, match=msg + "; letterboxing needs at least 2 pixels on each side"):
            api._check(_call(net, which, *size)[0])
    finally:
        net.set_letterbox(False)


@pytest.mark.parametrize("size", list(THIN), ids=[f"{w}x{h}" for w, h in THIN])
@pytest.mark.parametrize("which", CALLS)
def test_thin_frames_pass_the_checks_with_letterbox_off(net, which, size):
    """Stretched, the same frames are valid: the call either runs (on a GPU) or fails later for a reason that is not the
    letterbox (no device here; the dummy device-frame pointer is not device memory)."""
    from yolo2_light_b200 import api
    ok, t = _call(net, which, *size)
    if ok and which.startswith("submit"):
        rows, counts = C.POINTER(C.c_float)(), C.POINTER(C.c_int)()
        assert api.lib().yb_network_collect_detections(net._h, t, 0, C.byref(rows), C.byref(counts), None) > 0
    if not ok:
        err = api.lib().yb_last_error().decode()
        assert "letterbox" not in err, err
        if which.endswith("device_frames"):
            assert "frame 0 is" in err, err


def test_frame_that_fits_is_accepted_by_the_checks(net):
    """640 x 20 letterboxes to 64 x 2, the smallest height the resize takes."""
    from yolo2_light_b200 import api
    net.set_letterbox(True)
    try:
        ok, _ = _call(net, "predict_frames_u8", 640, 20)
        assert ok or "letterbox" not in api.lib().yb_last_error().decode()
    finally:
        net.set_letterbox(False)
