"""The detector's drawing (draw_detections_v3 of test_detector, src/main.c:38-148) with the reference library's own
draw_box_width and get_color (tests/draw_ref.py) against its full numpy restatement (tests/draw_util.py), on synthetic
detection sets: boxes partly or wholly
outside the frame, boxes narrower than two line widths and crossing rectangles, frames below 167 rows (line width 1),
1, 80 and 601 classes, equal probabilities and equal left edges, a probability exactly at thresh, and non-finite and
out-of-int coordinates."""
import numpy as np
import pytest

import draw_ref
import draw_util
import ybtest_util as util

needs_ref = pytest.mark.skipif(not util.have_ref(), reason="reference build absent")

# (w, h): line width 1 (h < 167), 1 at h = 166, 2 at 334, and a 1-pixel frame
SIZES = [(64, 48), (200, 166), (97, 167), (300, 334), (1, 1), (5, 400)]


@needs_ref
@pytest.mark.parametrize("classes", [1, 80, 601])
@pytest.mark.parametrize("size", SIZES)
def test_reference_drawing_equals_restatement(classes, size):
    w, h = size
    rng = np.random.default_rng(classes * 1000 + w + h)
    thresh = 0.25
    rows = draw_util.synthetic_rows(rng, 60, classes, thresh)
    frame = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    got, lr, lc = draw_ref.draw_detections(frame, rows, classes, thresh)
    exp, er, ec = draw_util.draw_detections(frame, rows, classes, thresh)
    assert list(lr) == er and list(lc) == ec
    assert np.array_equal(got, exp)
    assert 6 not in er                              # its probability equals thresh
    assert {0, 1, 2, 3, 7, 8, 9, 10, 11} <= set(er)   # equal keys, NaN, inf and out-of-int boxes are selected and drawn


def test_equal_keys_keep_candidate_order():
    classes = 3
    rows = np.zeros((5, 8), np.float32)
    rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3] = [0.5, 0.5, 0.3, 0.5, 0.5], 0.5, [0.2, 0.2, 0.2, 0.2, 0.2], 0.2
    rows[:, 5 + 1] = [0.6, 0.6, 0.6, 0.7, 0.6]
    lr, lc, dr, dc = draw_util.select(rows, classes, 0.5)
    assert list(lr) == [2, 0, 1, 3, 4] and list(dr) == [0, 1, 2, 4, 3] and set(lc) == {1}


@needs_ref
def test_drawn_bytes_of_undrawn_pixels_are_unchanged():
    """u8 -> /255. -> x255 -> truncation gives every byte back, so a frame without boxes comes back as it went in."""
    frame = np.arange(256 * 3, dtype=np.int64).reshape(16, 16, 3).astype(np.uint8)
    assert np.array_equal(draw_ref.draw_boxes(frame, np.zeros((0, 4), np.float32), np.zeros(0, np.int32), 80), frame)
    v = np.arange(256, dtype=np.float32)
    assert np.array_equal((np.float32(255) * (v / np.float64(255.)).astype(np.float32)).astype(np.int64), np.arange(256))


@needs_ref
def test_colours_of_every_class_match_the_reference():
    for classes in (1, 2, 80, 601):
        cls = np.arange(classes, dtype=np.int32)
        boxes = np.tile(np.float32([[0.5, 0.5, 0.0, 0.0]]), (classes, 1))
        frame = np.zeros((1, 1, 3), np.uint8)
        for c in cls[:: max(1, classes // 97)]:
            got = draw_ref.draw_boxes(frame, boxes[c:c + 1], cls[c:c + 1], classes)
            assert tuple(got[0, 0]) == draw_util.colour(int(c), classes), (classes, c)
