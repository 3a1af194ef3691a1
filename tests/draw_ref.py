"""The reference's own drawing functions, called through ctypes on the reference library the oracle build makes
(oracle/_ref/libyolo2ref_scalar.so, which exports draw_box_width, get_color, make_image and free_image from
src/additionally.c).  draw_detections_v3 itself lives in src/main.c, which that library does not compile, so its selection,
its two orders and its corner arithmetic (main.c:38-143) come from the restatement in tests/draw_util.py; the rectangles,
the colours and the float image they are drawn into are the reference's."""
import ctypes as C

import numpy as np

import draw_util


class Image(C.Structure):
    """``image`` of src/additionally.h:837-842"""
    _fields_ = [("h", C.c_int), ("w", C.c_int), ("c", C.c_int), ("data", C.POINTER(C.c_float))]


_lib = None


def _load():
    global _lib
    if _lib is None:
        from oracle import ref
        L = C.CDLL(ref.lib_path("scalar"))
        L.draw_box_width.restype = None
        L.draw_box_width.argtypes = [Image, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
        L.get_color.restype = C.c_float
        L.get_color.argtypes = [C.c_int, C.c_int, C.c_int]
        _lib = L
    return _lib


def get_color(c, x, mx):
    return _load().get_color(c, x, mx)


def draw_boxes(rgb, boxes, cls, classes):
    """boxes [n, 4] (relative x, y, w, h) with best classes cls[n] drawn in the given order into a copy of the u8 RGB frame
    [h, w, 3] by the reference's draw_box_width and get_color, as draw_detections_v3 draws them (main.c:107-143); the float
    image is built as load_image_stb builds it (additionally.c:3093-3103) and written back as save_image_png writes it
    (additionally.c:3226)."""
    L = _load()
    img = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = img.shape
    data = np.ascontiguousarray((img.transpose(2, 0, 1).astype(np.float64) / 255.).astype(np.float32))
    im = Image(h, w, 3, data.ctypes.data_as(C.POINTER(C.c_float)))
    width = max(1, int(h * .006))                                   # main.c:109-111
    for box, c in zip(np.asarray(boxes, np.float32).reshape(-1, 4), cls):
        offset = int(c) * 123457 % classes                          # main.c:116
        red, green, blue = (L.get_color(k, offset, classes) for k in (2, 1, 0))
        left, top, right, bot = draw_util.corners(box, w, h)        # main.c:125-133
        L.draw_box_width(im, left, top, right, bot, width, red, green, blue)
    return (np.float32(255) * data).astype(np.int32).astype(np.uint8).transpose(1, 2, 0).copy()


def draw_detections(rgb, rows, classes, thresh):
    """draw_detections_v3 of test_detector on one image's rows [n, 5 + classes] (relative boxes): (drawn u8 RGB frame,
    selected rows in list order, their classes)."""
    rows = np.asarray(rows, np.float32).reshape(-1, 5 + classes)
    lp, lc, dp, dc = draw_util.select(rows, classes, thresh)
    boxes = rows[dp, :4] if dp else np.zeros((0, 4), np.float32)
    return draw_boxes(rgb, boxes, dc, classes), lp, lc
