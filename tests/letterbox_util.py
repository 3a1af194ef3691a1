"""Helpers of the letterbox tests: darknet's letterbox_image (resize_image to the letterbox size, fill_image(.5),
embed_image) built two ways -- on the oracle's restatement of the resize (oracle/port.load_resize_u8), and on the
unmodified reference's own make_image / resize_image called through ctypes -- and the reference's get_network_boxes with
its `letter` argument.  The reference has no letterbox_image (its loader stubs LETTERBOX_DATA, additionally.c:4418-4422),
so the fill and the embed are written here, in numpy."""
import ctypes as C

import numpy as np


# (w, h) -> (nw, nh, dx, dy) in a 64 x 64 network: wide, tall, already its letterbox size, the network's aspect ratio,
# an upscale with an odd margin, a target height of 2, and rows wider than the resize kernel stages in shared memory
LETTERBOX_CASES = {
    (640, 480): (64, 48, 0, 8),
    (100, 300): (21, 64, 21, 0),
    (64, 36): (64, 36, 0, 14),
    (128, 128): (64, 64, 0, 0),
    (35, 17): (64, 31, 0, 16),
    (640, 20): (64, 2, 0, 31),
    (4500, 400): (64, 5, 0, 29),
}
SIZES = list(LETTERBOX_CASES)


def letterbox_size(netw, neth, w, h):
    """correct_yolo_boxes' integer letterbox size (additionally.c:4287-4294), the float compare done in float32 as C does."""
    if np.float32(netw) / np.float32(w) < np.float32(neth) / np.float32(h):
        return netw, (h * netw) // w
    return (w * neth) // h, neth


def _embed(resized, out_w, out_h):
    """resized float32[c, nh, nw] centred on an out_w x out_h canvas of 0.5 at ((out_w - nw) / 2, (out_h - nh) / 2)."""
    c, nh, nw = resized.shape
    out = np.full((c, out_h, out_w), 0.5, np.float32)
    dx, dy = (out_w - nw) // 2, (out_h - nh) // 2
    out[:, dy:dy + nh, dx:dx + nw] = resized
    return out


def port_letterbox_u8(img_hwc, out_w, out_h):
    """letterbox_image on the oracle's restatement of load_image_stb + resize_image -> float32[c, out_h, out_w]."""
    from oracle import port
    h, w, _ = img_hwc.shape
    nw, nh = letterbox_size(out_w, out_h, w, h)
    return _embed(port.load_resize_u8(img_hwc, nw, nh), out_w, out_h)


class _Image(C.Structure):   # the reference's image (additionally.h:837-842)
    _fields_ = [("h", C.c_int), ("w", C.c_int), ("c", C.c_int), ("data", C.POINTER(C.c_float))]


class _Box(C.Structure):     # box.h:4-6
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("w", C.c_float), ("h", C.c_float)]


class _Detection(C.Structure):   # box.h:9-16
    _fields_ = [("bbox", _Box), ("classes", C.c_int), ("prob", C.POINTER(C.c_float)), ("mask", C.POINTER(C.c_float)),
                ("objectness", C.c_float), ("sort_class", C.c_int)]


def _ref_lib():
    from oracle import ref
    L = ref._load("scalar")
    L.make_image.restype = _Image
    L.make_image.argtypes = [C.c_int, C.c_int, C.c_int]
    L.resize_image.restype = _Image
    L.resize_image.argtypes = [_Image, C.c_int, C.c_int]
    L.free_image.restype = None
    L.free_image.argtypes = [_Image]
    L.get_network_boxes.restype = C.POINTER(_Detection)
    L.get_network_boxes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_int,
                                    C.POINTER(C.c_int), C.c_int]
    L.do_nms_sort.restype = None
    L.do_nms_sort.argtypes = [C.POINTER(_Detection), C.c_int, C.c_int, C.c_float]
    L.free_detections.restype = None
    L.free_detections.argtypes = [C.POINTER(_Detection), C.c_int]
    return L


def ref_letterbox_u8(img_hwc, out_w, out_h):
    """letterbox_image on the reference: load_image_stb's conversion ((float)byte / 255. in double, additionally.c:3100)
    into the reference's make_image, its resize_image to the letterbox size, then the fill and the embed."""
    L = _ref_lib()
    img = np.ascontiguousarray(img_hwc, dtype=np.uint8)
    h, w, c = img.shape
    nw, nh = letterbox_size(out_w, out_h, w, h)
    im = L.make_image(w, h, c)
    planar = np.ascontiguousarray((img.transpose(2, 0, 1).astype(np.float64) / 255.).astype(np.float32))
    C.memmove(im.data, planar.ctypes.data, planar.nbytes)
    resized = L.resize_image(im, nw, nh)
    try:
        r = np.ctypeslib.as_array(resized.data, shape=(c, nh, nw)).copy()
    finally:
        L.free_image(resized)
        L.free_image(im)
    return _embed(r, out_w, out_h)


def ref_boxes(rnet, w, h, thresh, nms, letter):
    """The reference's get_network_boxes(net, w, h, thresh, .5, NULL, relative = 1, &n, letter) + do_nms_sort after
    rnet.predict: rows {x, y, w, h, objectness, prob[0..classes)} (the row format of the device decode)."""
    L = _ref_lib()
    classes = rnet.layers[-1]["classes"]
    n = C.c_int()
    dets = L.get_network_boxes(C.c_void_p(rnet.h), w, h, thresh, 0.5, None, 1, C.byref(n), letter)   # refh starts with its network
    try:
        if nms > 0:
            L.do_nms_sort(dets, n.value, classes, nms)
        out = np.zeros((n.value, 5 + classes), np.float32)
        for k in range(n.value):
            d = dets[k]
            out[k, :5] = (d.bbox.x, d.bbox.y, d.bbox.w, d.bbox.h, d.objectness)
            out[k, 5:] = np.ctypeslib.as_array(d.prob, shape=(classes,))
    finally:
        L.free_detections(dets, n.value)
    return out
