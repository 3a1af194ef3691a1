"""Helpers of the drawing tests: draw_detections_v3 of the reference's test_detector (src/main.c:38-148, draw_box_width /
draw_box / get_color of src/additionally.c) restated in numpy, for RGB frames and for the NV12 rule of
yb_network_submit_device_frames_draw, and synthetic detection rows."""
import math

import numpy as np

INF = float("inf")
COLORS = np.array([[1, 0, 1], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 1, 0], [1, 0, 0]], np.float32)


def select(rows, classes, thresh):
    """get_actual_detections and the two orders: (list_pos, list_cls, draw_pos, draw_cls) of one image's rows
    [n, 5 + classes]; equal keys in candidate order, a NaN left edge as +inf."""
    rows = np.asarray(rows, np.float32).reshape(-1, 5 + classes)
    thresh = np.float32(thresh)
    pos, cls = [], []
    for i, r in enumerate(rows):
        best, bp = -1, thresh
        for j in range(classes):
            if r[5 + j] > bp:
                best, bp = j, r[5 + j]
        if best >= 0:
            pos.append(i)
            cls.append(best)
    left = [float(rows[p, 0] - rows[p, 2] / np.float32(2)) for p in pos]
    left = [INF if k != k else k for k in left]
    lo = sorted(range(len(pos)), key=lambda k: (left[k], pos[k]))
    do = sorted(range(len(pos)), key=lambda k: (float(rows[pos[k], 5 + cls[k]]), pos[k]))
    return ([pos[k] for k in lo], [cls[k] for k in lo], [pos[k] for k in do], [cls[k] for k in do])


def d2i(v):
    """x86 cvttsd2si: truncation, INT_MIN for NaN and out-of-int values"""
    return math.trunc(v) if -2147483649.0 < v < 2147483648.0 else -2 ** 31


def wrap(v):
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


def get_color(c, x, mx):
    ratio = np.float32(np.float32(x) / np.float32(mx)) * np.float32(5)
    i, j = math.floor(float(ratio)), math.ceil(float(ratio))
    ratio = np.float32(ratio - np.float32(i))
    return np.float32(np.float32((np.float32(1) - ratio) * COLORS[i, c]) + np.float32(ratio * COLORS[j, c]))


def colour(cls, classes):
    """the (r, g, b) bytes of a class, as save_image_png writes get_color's floats"""
    assert cls * 123457 < 2 ** 31
    off = cls * 123457 % classes
    return tuple(int(np.float32(255) * get_color(2 - k, off, classes)) for k in range(3))


def rgb_to_yuv(r, g, b):
    """the BT.601 limited-range integer rule of include/yolo2_light_b200.h (YB_FRAME_NV12)"""
    return (((66 * r + 129 * g + 25 * b + 128) >> 8) + 16, ((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128,
            ((112 * r - 94 * g - 18 * b + 128) >> 8) + 128)


def corners(box, w, h):
    """draw_detections_v3's left, top, right, bot of a relative box (x, y, w, h), main.c:125-133"""
    x, y, bw, bh = (float(np.float32(v)) for v in box)
    left, right = d2i((x - bw / 2.) * w), d2i((x + bw / 2.) * w)
    top, bot = d2i((y - bh / 2.) * h), d2i((y + bh / 2.) * h)
    return max(left, 0), max(top, 0), right if right <= w - 1 else w - 1, bot if bot <= h - 1 else h - 1


def box_pixels(left, top, right, bot, w, h):
    """the (ys, xs) index arrays draw_box_width touches, in any order"""
    width = max(1, int(h * .006))
    ys, xs = [], []
    for i in range(width):
        x1, y1, x2, y2 = wrap(left + i), wrap(top + i), wrap(right - i), wrap(bot - i)
        x1, x2 = min(max(x1, 0), w - 1), min(max(x2, 0), w - 1)
        y1, y2 = min(max(y1, 0), h - 1), min(max(y2, 0), h - 1)
        if x2 >= x1:
            xr = np.arange(x1, x2 + 1)
            xs += [xr, xr]
            ys += [np.full_like(xr, y1), np.full_like(xr, y2)]
        if y2 >= y1:
            yr = np.arange(y1, y2 + 1)
            ys += [yr, yr]
            xs += [np.full_like(yr, x1), np.full_like(yr, x2)]
    if not xs:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(ys), np.concatenate(xs)


def draw_rgb(frame, boxes, cls, classes):
    """boxes [n, 4] with classes cls[n] drawn in the given order into a copy of the u8 RGB frame [h, w, 3]"""
    out = np.array(frame, np.uint8, copy=True)
    h, w, _ = out.shape
    for box, c in zip(boxes, cls):
        ys, xs = box_pixels(*corners(box, w, h), w, h)
        out[ys, xs] = colour(int(c), classes)
    return out


def draw_nv12(nv12, boxes, cls, classes):
    """the same boxes drawn into a copy of an NV12 frame [3h/2, w]: each drawn pixel's Y, and the U, V of every 2x2 block
    with a drawn pixel from the last box (in the given order) that covers one"""
    out = np.array(nv12, np.uint8, copy=True)
    h, w = out.shape[0] // 3 * 2, out.shape[1]
    for box, c in zip(boxes, cls):
        ys, xs = box_pixels(*corners(box, w, h), w, h)
        Y, U, V = rgb_to_yuv(*colour(int(c), classes))
        out[ys, xs] = Y
        out[h + ys // 2, xs & ~1] = U
        out[h + ys // 2, (xs & ~1) + 1] = V
    return out


def draw_detections(frame, rows, classes, thresh, nv12=False):
    """draw_detections_v3 of one image: (drawn frame, list positions, list classes)"""
    rows = np.asarray(rows, np.float32).reshape(-1, 5 + classes)
    lp, lc, dp, dc = select(rows, classes, thresh)
    boxes = rows[dp, :4] if dp else np.zeros((0, 4), np.float32)
    return (draw_nv12 if nv12 else draw_rgb)(frame, boxes, dc, classes), lp, lc


def synthetic_rows(rng, n, classes, thresh, special=True):
    """n candidate rows {x, y, w, h, objectness, prob[classes]} with relative boxes: many inside the frame, some partly or
    wholly outside, narrow and crossing ones, equal probabilities and equal left edges, probabilities exactly at thresh, and
    non-finite and out-of-int coordinates"""
    rows = np.zeros((n, 5 + classes), np.float32)
    rows[:, 0] = rng.uniform(-0.3, 1.3, n)
    rows[:, 1] = rng.uniform(-0.3, 1.3, n)
    rows[:, 2] = rng.uniform(0, 0.8, n) ** 2
    rows[:, 3] = rng.uniform(0, 0.8, n) ** 2
    rows[:, 4] = 1
    k = rng.integers(0, classes, (n, 3))
    for i in range(n):
        for j in k[i]:
            rows[i, 5 + j] = rng.choice([rng.uniform(0, 1), thresh, 0.5, 0.75])
    if special and n >= 12:
        rows[[0, 2, 3], 5 + k[[0, 2, 3], 0]] = 0.6
        rows[1, :4] = rows[0, :4]                     # the same box twice
        rows[1, 5:] = rows[0, 5:]                     # with equal probabilities
        rows[2, 0], rows[2, 2] = rows[3, 0], rows[3, 2]   # equal left edges
        rows[4, 2] = rows[4, 3] = 0                   # a point
        rows[5, 2], rows[5, 3] = 0.001, 0.5           # narrower than two line widths
        rows[6, 5:] = 0
        rows[6, 5 + k[6, 0]] = thresh                 # exactly at thresh: not selected
        rows[7, 0] = np.nan                           # NaN coordinates
        rows[8, 2] = np.inf                           # an infinite width
        rows[9, 0] = 3e9                              # outside int after scaling
        rows[10, 1] = -3e9
        rows[11, 3] = 1e30
        for i in range(6, 12):
            if i != 6:
                rows[i, 5 + k[i, 0]] = 0.9
    return rows
