"""Drawing each image's detections into its device frame (yb_network_submit_device_frames_draw): the rows and counts are
those of yb_network_submit_device_frames; RGB frames come out bit for bit as the reference's draw_detections_v3 draws the
ticket's own rows (with the reference library's draw_box_width and get_color, tests/draw_ref.py, or its numpy
restatement in tests/draw_util.py where the reference build is absent), with the row padding and every uncovered pixel untouched; BGR and planar frames are that result permuted; NV12
frames follow the NV12 rule; the selected list is the oracle's; and the caller's stream sees the drawn frames."""
import numpy as np
import pytest

import draw_util
import ybtest_util as util
from device_frames_util import device_frame, random_frame

pytestmark = pytest.mark.gpu

# mixed sizes with odd ones, a 1-pixel frame and a partial batch
RGB_SETS = [[(120, 97), (64, 64), (33, 201)], [(301, 170)], [(64, 64), (1, 1)], [(250, 333), (7, 5), (640, 168)]]
NV12_SETS = [[(120, 96), (64, 64), (34, 200)], [(300, 170)], [(2, 2), (640, 168)]]


def _oracle(frame, rows, classes, thresh):
    if util.have_ref():
        import draw_ref
        return draw_ref.draw_detections(frame, rows, classes, thresh)
    return draw_util.draw_detections(frame, rows, classes, thresh)


def _storage(t):
    """all bytes of a tensor's storage, on the host"""
    import torch
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage()).cpu().numpy()


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    import yolo2_light_b200 as yb
    wd = str(tmp_path_factory.mktemp("draw"))
    tiny, q = util.mixed_net("tiny64_fp32", wd)
    s2, _ = util.mixed_net("s2chain", wd)
    cfg, wts = util.bigger("tiny", wd, 256, 256)
    big = util.load(cfg, wts, 3, precision=yb.YB_PREC_BF16_TC)
    return {"tiny64": (tiny, 0.05), "s2chain": (s2, 0.05), "tiny256": (big, 0.05)}


def _plain_and_draw(net, dev, fmt, thresh, letter, max_rows=4096):
    t = net.submit_device_frames(dev, thresh, fmt=fmt, relative=1, letter=letter, max_rows=max_rows)
    rows0, cnt0, moved0 = net.collect_detections(t)
    t = net.submit_device_frames_draw(dev, thresh, fmt=fmt, letter=letter, max_rows=max_rows)
    assert net.selected_detections(t) is None          # not collected yet
    rows1, cnt1, moved1 = net.collect_detections(t)
    sel = net.selected_detections(t)
    assert np.array_equal(cnt0, cnt1)
    for a, b in zip(rows0, rows1):
        assert util.bits_equal(a, b)
    nsel = sum(len(s) for s in sel)
    assert moved1 == moved0 + 4 * net.batch + 28 * nsel
    return rows1, sel


def _check_list(sel, rows, lr, lc):
    assert list(sel["row"]) == lr and list(sel["cls"]) == lc
    if lr:
        r = rows[lr]
        assert util.bits_equal(np.stack([sel["x"], sel["y"], sel["w"], sel["h"]], 1), r[:, :4])
        assert util.bits_equal(sel["prob"], r[np.arange(len(lr)), 5 + np.array(lc)])


@pytest.mark.parametrize("layout", ["padded", "odd_offset"])
@pytest.mark.parametrize("letter", [0, 1])
@pytest.mark.parametrize("kind", ["tiny64", "s2chain", "tiny256"])
def test_rgb_frames_equal_the_reference_drawing(nets, kind, letter, layout):
    net, thresh = nets[kind]
    classes = net.layer(net.n - 1)["classes"]
    rng = np.random.default_rng(11 + 3 * letter + len(kind))
    net.set_letterbox(bool(letter))
    try:
        drawn = []
        for sizes in RGB_SETS:
            frames = [random_frame("rgb", w, h, rng) for w, h in sizes]
            dev = [device_frame("rgb", f, layout) for f in frames]
            rows, sel = _plain_and_draw(net, dev, "rgb", thresh, letter)
            for b, f in enumerate(frames):
                exp, lr, lc = _oracle(f, rows[b], classes, thresh)
                want = _storage(device_frame("rgb", exp, layout, device="cpu"))
                got = _storage(dev[b])
                assert np.array_equal(got, want), (kind, letter, layout, sizes, b)
                _check_list(sel[b], rows[b], lr, lc)
                drawn.append(len(lr))
    finally:
        net.set_letterbox(False)
    assert sum(drawn) > 0
    if kind != "tiny64":
        assert max(drawn) >= 100, drawn            # hundreds of overlapping boxes in one frame


@pytest.mark.parametrize("fmt", ["bgr", "planar"])
def test_bgr_and_planar_frames_are_the_rgb_result_permuted(nets, fmt):
    net, thresh = nets["tiny256"]
    classes = net.layer(net.n - 1)["classes"]
    rng = np.random.default_rng(5)
    for sizes in RGB_SETS[:3]:
        rgb = [random_frame("rgb", w, h, rng) for w, h in sizes]
        frames = [f[..., ::-1].copy() if fmt == "bgr" else f.transpose(2, 0, 1).copy() for f in rgb]
        dev = [device_frame(fmt, f, "padded") for f in frames]
        rows, sel = _plain_and_draw(net, dev, fmt, thresh, 0)
        for b, f in enumerate(rgb):
            exp, lr, lc = _oracle(f, rows[b], classes, thresh)
            exp = exp[..., ::-1].copy() if fmt == "bgr" else exp.transpose(2, 0, 1).copy()
            assert np.array_equal(_storage(dev[b]), _storage(device_frame(fmt, exp, "padded", device="cpu"))), (sizes, b)
            _check_list(sel[b], rows[b], lr, lc)


@pytest.mark.parametrize("layout", ["padded", "tight"])
def test_nv12_frames_follow_the_nv12_rule(nets, layout):
    net, thresh = nets["tiny256"]
    classes = net.layer(net.n - 1)["classes"]
    rng = np.random.default_rng(9)
    for sizes in NV12_SETS:
        frames = [random_frame("nv12", w, h, rng) for w, h in sizes]
        dev = [device_frame("nv12", f, layout) for f in frames]
        rows, sel = _plain_and_draw(net, dev, "nv12", thresh, 0)
        for b, f in enumerate(frames):
            lr, lc, dr, dc = draw_util.select(rows[b], classes, thresh)
            exp = draw_util.draw_nv12(f, rows[b][dr, :4] if dr else np.zeros((0, 4), np.float32), dc, classes)
            assert np.array_equal(_storage(dev[b]), _storage(device_frame("nv12", exp, layout, device="cpu"))), (sizes, b)
            _check_list(sel[b], rows[b], lr, lc)


def test_callers_stream_sees_the_drawn_frames(nets):
    """Frames written on the caller's stream behind a delay, the draw call, then a copy of the frames on the same stream
    right after the call, with no synchronisation: the copy holds the drawn frames."""
    import torch
    net, thresh = nets["tiny256"]
    classes = net.layer(net.n - 1)["classes"]
    rng = np.random.default_rng(21)
    sizes = [(320, 240), (97, 131), (640, 360)]
    frames = [random_frame("rgb", w, h, rng) for w, h in sizes]
    dev = [device_frame("rgb", np.zeros_like(f), "padded") for f in frames]
    src = [torch.from_numpy(f).cuda() for f in frames]
    copies = [torch.empty_like(d) for d in dev]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        for d, x in zip(dev, src):
            d.copy_(x)
        t = net.submit_device_frames_draw(dev, thresh, fmt="rgb", max_rows=4096, stream=s.cuda_stream)
        for c, d in zip(copies, dev):
            c.copy_(d)
    rows, _, _ = net.collect_detections(t)
    torch.cuda.synchronize()
    n = 0
    for b, f in enumerate(frames):
        exp, lr, _ = _oracle(f, rows[b], classes, thresh)
        assert np.array_equal(copies[b].cpu().numpy(), exp), b
        n += len(lr)
    assert n > 0


def test_selected_list_lifetime(nets):
    """The list is there from the collect until the slot is taken again, and only for drawing tickets."""
    import torch
    net, thresh = nets["tiny64"]
    rng = np.random.default_rng(3)
    dev = [device_frame("rgb", random_frame("rgb", 64, 64, rng), "tight") for _ in range(3)]
    t = net.submit_device_frames_draw(dev, thresh, fmt="rgb", max_rows=256)
    net.collect_detections(t)
    first = net.selected_detections(t)
    assert first is not None and len(first) == 3
    assert all(np.array_equal(a, b) for a, b in zip(first, net.selected_detections(t)))
    others = []
    for _ in range(2):   # the other two slots
        others.append(net.submit_device_frames(dev, thresh, fmt="rgb", max_rows=256))
        net.collect_detections(others[-1])
    assert all(net.selected_detections(o) is None for o in others)
    assert net.selected_detections(t) is not None
    t2 = net.submit_device_frames(dev, thresh, fmt="rgb", max_rows=256)   # slot of t again
    assert t2 == t and net.selected_detections(t) is None
    net.collect_detections(t2)
    assert net.selected_detections(t) is None
    torch.cuda.synchronize()
