"""The letterbox input of darknet's letterbox_image on the CPU: built on the oracle's restatement of the resize against
the same built on the unmodified reference's make_image + resize_image (letterbox_util), bit for bit, and the geometry of
the restatement: where the image lies and that the band around it is 0.5."""
import numpy as np
import pytest

import ybtest_util as util
from letterbox_util import LETTERBOX_CASES, SIZES, letterbox_size, port_letterbox_u8, ref_letterbox_u8

NET = 64


def _frame(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_port_letterbox_geometry(size):
    from oracle import port
    w, h = size
    nw, nh, dx, dy = LETTERBOX_CASES[size]
    assert letterbox_size(NET, NET, w, h) == (nw, nh)
    f = _frame(w, h, 11 + w + h)
    got = port_letterbox_u8(f, NET, NET)
    assert got.shape == (3, NET, NET)
    inside = got[:, dy:dy + nh, dx:dx + nw]
    assert util.bits_equal(inside, port.load_resize_u8(f, nw, nh))
    band = np.ones((NET, NET), bool)
    band[dy:dy + nh, dx:dx + nw] = False
    assert np.all(got[:, band] == np.float32(0.5))


@pytest.mark.skipif(not util.have_ref(), reason="reference build absent")
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_port_letterbox_equals_reference(size):
    w, h = size
    f = _frame(w, h, 23 + w * h)
    assert util.bits_equal(port_letterbox_u8(f, NET, NET), ref_letterbox_u8(f, NET, NET)), size


@pytest.mark.skipif(not util.have_ref(), reason="reference build absent")
def test_port_letterbox_equals_reference_non_square_network():
    """A 96 x 64 network: the limiting side and the offsets swap with the frame's shape."""
    for k, (w, h) in enumerate([(640, 480), (100, 300), (96, 64), (50, 51), (30, 200)]):
        f = _frame(w, h, 300 + k)
        assert util.bits_equal(port_letterbox_u8(f, 96, 64), ref_letterbox_u8(f, 96, 64)), (w, h)


@pytest.mark.skipif(not util.have_ref(), reason="reference build absent")
def test_reference_boxes_helper_equals_harness(tmp_path):
    """The ctypes call of get_network_boxes in letterbox_util gives, at letter = 0, the harness's own rows (refh_get_boxes)
    with its sort_class column dropped; at letter = 1 for a non-square frame the boxes move, the scores do not."""
    from oracle import ref
    from letterbox_util import ref_boxes
    cfg, wts = util.model_files("tiny64", str(tmp_path))
    rnet = ref.RefNet(cfg, wts, 1, 0, 7)
    rnet.predict(port_letterbox_u8(_frame(640, 480, 5), NET, NET)[None])
    mine = ref_boxes(rnet, 640, 480, 0.2, 0.45, 0)
    theirs = np.delete(rnet.get_boxes(640, 480, 0.2, 0.45), 5, axis=1)
    assert mine.shape[0] > 0 and util.bits_equal(mine, theirs)
    lb = ref_boxes(rnet, 640, 480, 0.2, 0.45, 1)
    assert lb.shape == mine.shape and util.bits_equal(lb[:, 4:], mine[:, 4:]) and not util.bits_equal(lb[:, :4], mine[:, :4])
