"""Letterboxed frames on the device (yb_network_set_letterbox): the input k_resize_frames makes equals darknet's
letterbox_image (on the oracle's restatement of the resize, pinned against the reference in test_letterbox_oracle.py) for host frames of
mixed sizes and partial batches; device frames of every format give what their host frames give; frames of the network's
aspect ratio give the same input and detections with letterboxing on and off; boxes with letter = 1 match the unmodified
reference run on its own letterboxed input; and the pipelined calls equal the synchronous ones.  Comparisons are bitwise
unless stated otherwise."""
import numpy as np
import pytest

import ybtest_util as util
from device_frames_util import device_frame, equivalent_host_frame, random_frame
from letterbox_util import SIZES, port_letterbox_u8, ref_boxes, ref_letterbox_u8
from ybtest_util import bigger, mixed_net, sorted_rows

pytestmark = pytest.mark.gpu

FORMATS = ["rgb", "bgr", "planar", "nv12"]
# the letterbox size list of test_letterbox_oracle.py in mixed and partial batches of 4
HOST_SETS = [[(640, 480), (100, 300), (64, 36), (128, 128)],
             [(35, 17), (640, 20), (4500, 400)],
             [(100, 300)]]
# its even sizes, for NV12
EVEN_SETS = [[(640, 480), (100, 300), (64, 36), (128, 128)],
             [(640, 20), (4500, 400)]]


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    import yolo2_light_b200 as yb
    net = util.load(*util.model_files("tiny64", str(tmp_path_factory.mktemp("letterbox"))), 4, precision=yb.YB_PREC_FP32)
    net.set_letterbox(True)
    return net


def test_size_list_covers_every_case():
    assert sorted(s for st in HOST_SETS for s in st) == sorted(SIZES + [(100, 300)])
    assert all(w % 2 == 0 and h % 2 == 0 for st in EVEN_SETS for w, h in st)


@pytest.mark.parametrize("k", range(len(HOST_SETS)))
def test_letterboxed_input_equals_oracle(tiny, k):
    frames = util.frames(HOST_SETS[k], 500 + k)
    tiny.predict_frames_u8(frames)
    got = tiny.fetch_input()
    for b, f in enumerate(frames):
        exp = port_letterbox_u8(f, tiny.w, tiny.h)
        assert util.bits_equal(got[b], exp), (k, b, f.shape)
    tail = got[len(frames):]
    assert tail.size == 0 or not tail.view(np.uint32).any()


def test_one_size_call_letterboxes(tiny):
    frames = np.stack(util.frames([(100, 300)] * tiny.batch, 77))
    tiny.predict_image_u8(frames)
    got = tiny.fetch_input()
    for b in range(tiny.batch):
        assert util.bits_equal(got[b], port_letterbox_u8(frames[b], tiny.w, tiny.h)), b


@pytest.mark.parametrize("k", range(len(EVEN_SETS)))
@pytest.mark.parametrize("fmt", FORMATS)
def test_device_frames_equal_host_path(tiny, fmt, k):
    rng = np.random.default_rng(600 + 7 * k + FORMATS.index(fmt))
    frames = [random_frame(fmt, w, h, rng) for w, h in EVEN_SETS[k]]
    tiny.predict_frames_u8([equivalent_host_frame(fmt, f) for f in frames])
    exp = tiny.fetch_input().copy()
    tiny.predict_device_frames([device_frame(fmt, f, "odd_offset") for f in frames], fmt=fmt)
    got = tiny.fetch_input()
    for b in range(len(frames)):
        assert util.bits_equal(got[b], exp[b]), (fmt, k, b, frames[b].shape)
    tail = got[len(frames):]
    assert tail.size == 0 or not tail.view(np.uint32).any()


ASPECT = [(64, 64), (128, 128), (32, 32)]


@pytest.mark.parametrize("kind", ["tiny64_q1", "s2chain"])
def test_network_aspect_frames_unchanged_by_letterbox(kind, workdir):
    """Frames of the network's aspect ratio letterbox to the network size at (0, 0): the input, the detection tensors and
    the pipelined rows (the 8-bit stem reads network-size batches directly on s2chain) are those of the stretched path."""
    net, q = mixed_net(kind, workdir)
    batches = [util.frames(ASPECT, 31), util.frames([(64, 64)] * 3, 32), util.frames([(64, 64), (32, 32)], 33)]
    res = {}
    for on in (False, True):
        net.set_letterbox(on)
        out = []
        for fr in batches:
            net.predict_frames_u8(fr, quantized=q)
            out.append(("input", net.fetch_input(quantized=q).copy()))
            out += [(i, o.copy()) for i, o in sorted(net.detection_outputs().items())]
            t = net.submit_frames_u8(fr, 0.3, 0.45, relative=0, letter=int(on), max_rows=2048, quantized=q)
            d, c, _ = net.collect_detections(t, quantized=q)
            out += [("counts", c.copy())] + [("rows", x.copy()) for x in d]
        res[on] = out
    net.set_letterbox(False)
    assert len(res[False]) == len(res[True])
    for (ka, a), (kb, b) in zip(res[False], res[True]):
        assert ka == kb, (ka, kb)
        assert np.array_equal(a, b) if ka == "counts" else util.bits_equal(a, b), (kind, ka)


@pytest.mark.skipif(not util.have_ref(), reason="reference build absent")
def test_letterboxed_detections_vs_reference_per_image(workdir):
    """Each frame through the unmodified reference (its resize_image to the letterbox size, network_predict_cpu,
    get_network_boxes(w, h, ..., letter = 1) + do_nms_sort) against one mixed, partial FP32 batch with letterboxing on and
    detect_frames(..., letter = 1); criteria of test_gpu_frames.py::test_detect_frames_vs_reference_per_image."""
    import yolo2_light_b200 as yb
    from oracle import ref
    cfg, wts = bigger("tiny", workdir, 160, 160)
    net = util.load(cfg, wts, 3, precision=yb.YB_PREC_FP32)
    net.set_letterbox(True)
    sizes = [(640, 480), (100, 300)]
    frames = util.frames(sizes, 45)
    net.predict_frames_u8(frames)
    dets, counts = net.detect_frames(sizes, 0.2, 0.45, letter=1, max_rows=4096)
    rnet = ref.RefNet(cfg, wts, 1, 0, 7)
    for b, ((w, h), f) in enumerate(zip(sizes, frames)):
        x = ref_letterbox_u8(f, rnet.width, rnet.height)
        assert util.bits_equal(net.fetch_input()[b], x), b
        rnet.predict(x[None])
        theirs = ref_boxes(rnet, w, h, 0.2, 0.45, 1)
        assert theirs.shape[0] > 0, b
        assert abs(int(counts[b]) - theirs.shape[0]) <= max(1, theirs.shape[0] // 100), (b, counts[b], theirs.shape)
        if counts[b] == theirs.shape[0] and theirs.shape[0]:
            a, e = sorted_rows(dets[b]), sorted_rows(theirs)
            assert np.allclose(a[:, :5], e[:, :5], rtol=1e-4, atol=1e-5)
            kept_a, kept_e = (a[:, 5:] > 0).sum(), (e[:, 5:] > 0).sum()
            assert abs(int(kept_a) - int(kept_e)) <= max(2, int(kept_e) // 50), (kept_a, kept_e)


# letterboxed, network-size (the direct stem path on s2chain, full and partial) and partial batches; all even for NV12
PIPE_BATCHES = [[(120, 96), (64, 64), (32, 200)], [(64, 64)] * 3, [(300, 170)], [(64, 64)] * 2, [(640, 480), (100, 300)],
                [(96, 96)] * 3, [(64, 36), (640, 20)]]


@pytest.mark.parametrize("kind", ["s2chain", "tiny64_q1"])
def test_pipelined_equal_sync_calls(kind, workdir):
    """submit_frames_u8 and submit_device_frames (formats in turn) with letterboxing on and letter = 1, three tickets in
    flight, against predict_frames_u8 / predict_device_frames + detect_frames."""
    net, q = mixed_net(kind, workdir)
    net.set_letterbox(True)
    thresh = 0.3
    rng = np.random.default_rng(41)
    fmts = [FORMATS[k % 4] for k in range(len(PIPE_BATCHES))]
    raw = [[random_frame(fmt, w, h, rng) for w, h in sizes] for fmt, sizes in zip(fmts, PIPE_BATCHES)]
    host = [[equivalent_host_frame(fmt, f) for f in fr] for fmt, fr in zip(fmts, raw)]
    dev = [[device_frame(fmt, f, "odd_offset") for f in fr] for fmt, fr in zip(fmts, raw)]

    def sync(k, device):
        if device:
            net.predict_device_frames(dev[k], fmt=fmts[k], quantized=q)
        else:
            net.predict_frames_u8(host[k], quantized=q)
        d, c = net.detect_frames(PIPE_BATCHES[k], thresh, 0.45, relative=0, letter=1, max_rows=2048, quantized=q)
        return [x.copy() for x in d], c.copy()

    def submit(k, device):
        if device:
            return net.submit_device_frames(dev[k], thresh, fmt=fmts[k], relative=0, letter=1, max_rows=2048, quantized=q)
        return net.submit_frames_u8(host[k], thresh, 0.45, relative=0, letter=1, max_rows=2048, quantized=q)

    total = 0
    for device in (False, True):
        exp = [sync(k, device) for k in range(len(PIPE_BATCHES))]
        total += sum(int(c.sum()) for _, c in exp)
        inflight, got = [], []
        for k in range(len(PIPE_BATCHES)):
            if len(inflight) == 3:
                got.append(net.collect_detections(inflight.pop(0), quantized=q)[:2])
            inflight.append(submit(k, device))
        while inflight:
            got.append(net.collect_detections(inflight.pop(0), quantized=q)[:2])
        for k, ((de, ce), (dg, cg)) in enumerate(zip(exp, got)):
            assert len(dg) == len(PIPE_BATCHES[k]) and np.array_equal(ce, cg), (kind, device, k, ce, cg)
            for b in range(len(de)):
                assert util.bits_equal(de[b], dg[b]), (kind, device, k, b)
    assert total > 0


def test_ticket_keeps_its_geometry(workdir):
    """The switch changes later calls only: a ticket submitted with letterboxing on and collected after it was turned off
    holds the letterboxed detections, and the next ticket the stretched ones."""
    net, q = mixed_net("tiny64_q1", workdir)
    fr = util.frames([(640, 480), (100, 300)], 55)
    sizes = [(640, 480), (100, 300)]
    exp = {}
    for on in (True, False):
        net.set_letterbox(on)
        net.predict_frames_u8(fr, quantized=q)
        d, c = net.detect_frames(sizes, 0.3, 0.45, relative=0, letter=int(on), max_rows=2048, quantized=q)
        exp[on] = ([x.copy() for x in d], c.copy())
    assert not np.array_equal(exp[True][1], exp[False][1]) or any(
        not util.bits_equal(a, b) for a, b in zip(exp[True][0], exp[False][0]))
    net.set_letterbox(True)
    t_on = net.submit_frames_u8(fr, 0.3, 0.45, relative=0, letter=1, max_rows=2048, quantized=q)
    net.set_letterbox(False)
    t_off = net.submit_frames_u8(fr, 0.3, 0.45, relative=0, letter=0, max_rows=2048, quantized=q)
    for t, on in ((t_on, True), (t_off, False)):
        d, c, _ = net.collect_detections(t, quantized=q)
        assert np.array_equal(c, exp[on][1]), on
        for b in range(len(d)):
            assert util.bits_equal(d[b], exp[on][0][b]), (on, b)
