"""Batches of frames of different sizes and partial batches: yb_network_predict_frames_u8, yb_network_detect_frames and
yb_network_submit_frames_u8.  Each image is resized and decoded on its own terms, as the reference app does per image
(src/main.c:188-229): the resized input equals the oracle's load_image + resize_image of that frame, a mixed batch
computes for each image what a batch of that frame alone computes, and each image's boxes are corrected for its own size.
Comparisons are bitwise unless stated otherwise."""
import os
import re

import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import INPUT_SETS, bigger, mixed_net, sorted_rows
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", range(len(INPUT_SETS)))
def test_resized_input_equals_reference_resize(k, workdir):
    import yolo2_light_b200 as yb
    from oracle import port
    net = util.load(*util.model_files("tiny64", workdir), 4, precision=yb.YB_PREC_FP32)
    frames = util.frames(INPUT_SETS[k], 100 + k)
    net.predict_frames_u8(frames)
    got = net.fetch_input()
    for b, f in enumerate(frames):
        exp = port.load_resize_u8(f, net.w, net.h)
        assert util.bits_equal(got[b], exp.reshape(got[b].shape)), (k, b, f.shape)
    tail = got[len(frames):]
    assert tail.size == 0 or np.array_equal(tail.view(np.uint32), np.zeros_like(tail.view(np.uint32)))


@pytest.mark.parametrize("kind", ["tiny64_fp32", "tiny64_bf16", "s2chain", "tiny64_q1", "xnor64"])
def test_no_leakage_across_images(kind, workdir):
    """Image b of a mixed batch gives the detection tensors a batch of that frame alone gives."""
    net, q = mixed_net(kind, workdir)
    frames = util.frames([(120, 96), (64, 64), (31, 200)], 7)
    net.predict_frames_u8(frames, quantized=q)
    mixed = {i: o.copy() for i, o in net.detection_outputs().items()}
    assert mixed
    for b, f in enumerate(frames):
        net.predict_image_u8(np.stack([f] * net.batch), quantized=q)
        for i, o in net.detection_outputs().items():
            assert util.bits_equal(mixed[i][b], o[b]), (kind, b, i)


SIZES = [(640, 480), (1280, 720), (333, 999)]


@pytest.mark.parametrize("relative,letter", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_detect_frames_equals_host_decode_per_image(relative, letter, workdir):
    B = 3
    net = util.load(*bigger("tiny", workdir, 160, 160), B)
    net.predict(cfgs.synthetic_images(B, 3, 160, 160, seed=43))
    for nimg in (3, 2):
        sizes = SIZES[:nimg]
        dets, counts = net.detect_frames(sizes, 0.2, 0.45, relative, letter, max_rows=4096)
        assert len(dets) == nimg and counts.shape == (nimg,)
        for b, (w, h) in enumerate(sizes):
            host = net.get_network_boxes(b, w, h, 0.2, 0.45, relative, letter)
            assert counts[b] == host.shape[0] > 0, (b, counts[b], host.shape)
            a, e = sorted_rows(dets[b]), sorted_rows(host)
            # boxes: double exp() on both sides, identical up to libm's last bit; probabilities: exact
            assert np.allclose(a[:, :4], e[:, :4], rtol=1e-6, atol=1e-7), b
            assert np.array_equal(a[:, 4:], e[:, 4:]), b
    # the C call writes counts[b] = 0 beyond nimg
    import ctypes as C
    from yolo2_light_b200 import api
    classes = net.layer_desc(net.n - 1).classes
    rows = np.zeros((B, 4096, 5 + classes), np.float32)
    cnt = np.full(B, -1, np.int32)
    ws, hs = (C.c_int * 1)(640), (C.c_int * 1)(480)
    r = api.lib().yb_network_detect_frames(net._h, 0, ws, hs, 1, 0.2, 0.45, relative, letter,
                                           rows.ctypes.data_as(C.c_void_p), 4096, cnt.ctypes.data_as(C.c_void_p))
    assert r == 5 + classes and cnt[0] > 0 and list(cnt[1:]) == [0, 0]


@pytest.mark.skipif(not util.have_ref(), reason="reference build absent")
def test_detect_frames_vs_reference_per_image(workdir):
    """Each frame through the unmodified reference (load_image + resize_image, forward, get_network_boxes + do_nms_sort for
    its own size) against one mixed, partial batch on the device in FP32; criteria of
    test_gpu_detect.py::test_device_detect_vs_reference_boxes."""
    import yolo2_light_b200 as yb
    from oracle import ref
    cfg, wts = bigger("tiny", workdir, 160, 160)
    net = util.load(cfg, wts, 3, precision=yb.YB_PREC_FP32)
    sizes = [(640, 480), (100, 300)]
    frames = util.frames(sizes, 45)
    net.predict_frames_u8(frames)
    dets, counts = net.detect_frames(sizes, 0.2, 0.45, max_rows=4096)
    rnet = ref.RefNet(cfg, wts, 1, 0, 7)
    for b, ((w, h), f) in enumerate(zip(sizes, frames)):
        rnet.predict(ref.load_resize_u8(f, rnet.width, rnet.height)[None])
        theirs = np.delete(rnet.get_boxes(w, h, 0.2, 0.45), 5, axis=1)
        assert abs(int(counts[b]) - theirs.shape[0]) <= max(1, theirs.shape[0] // 100), (b, counts[b], theirs.shape)
        if counts[b] == theirs.shape[0] and theirs.shape[0]:
            a, e = sorted_rows(dets[b]), sorted_rows(theirs)
            assert np.allclose(a[:, :5], e[:, :5], rtol=1e-4, atol=1e-5)
            kept_a, kept_e = (a[:, 5:] > 0).sum(), (e[:, 5:] > 0).sum()
            assert abs(int(kept_a) - int(kept_e)) <= max(2, int(kept_e) // 50), (kept_a, kept_e)


# batches of (w, h) per frame: varying nimg and sizes; on the 8-bit-stem net the network-size batches (64 x 64) take the
# direct stem path, once full and once partial
PIPE_BATCHES = [[(120, 96), (64, 64), (31, 200)], [(64, 64)] * 3, [(300, 170)], [(64, 64)] * 2, [(17, 23), (640, 480)],
                [(96, 96)] * 3, [(64, 64), (1, 1)]]


@pytest.mark.parametrize("kind", ["s2chain", "tiny64_q1"])
def test_pipelined_frames_equal_sync_calls(kind, workdir):
    net, q = mixed_net(kind, workdir)
    thresh = 0.3
    batches = [util.frames(sizes, 200 + k) for k, sizes in enumerate(PIPE_BATCHES)]
    exp = []
    for fr in batches:
        net.predict_frames_u8(fr, quantized=q)
        d, c = net.detect_frames([(f.shape[1], f.shape[0]) for f in fr], thresh, 0.45, relative=0, max_rows=2048, quantized=q)
        exp.append(([x.copy() for x in d], c.copy()))
    assert sum(int(c.sum()) for _, c in exp) > 0
    inflight, got = [], []
    for fr in batches:
        if len(inflight) == 3:
            d, c, _ = net.collect_detections(inflight.pop(0), quantized=q)
            got.append((d, c))
        inflight.append(net.submit_frames_u8(fr, thresh, 0.45, relative=0, max_rows=2048, quantized=q))
    while inflight:
        d, c, _ = net.collect_detections(inflight.pop(0), quantized=q)
        got.append((d, c))
    for k, ((de, ce), (dg, cg)) in enumerate(zip(exp, got)):
        assert len(dg) == len(PIPE_BATCHES[k]) and np.array_equal(ce, cg), (k, ce, cg)
        for b in range(len(de)):
            assert util.bits_equal(de[b], dg[b]), (k, b)


@pytest.mark.parametrize("fw,fh", [(64, 64), (120, 96)])
def test_uniform_frames_equal_submit_u8(fw, fh, workdir):
    net, q = mixed_net("s2chain", workdir)
    stacked = np.stack(util.frames([(fw, fh)] * net.batch, 9))
    t = net.submit_u8(stacked, 0.3, 0.45, relative=0, max_rows=2048)
    de, ce, me = net.collect_detections(t)
    t = net.submit_frames_u8(list(stacked), 0.3, 0.45, relative=0, max_rows=2048)
    dg, cg, mg = net.collect_detections(t)
    assert np.array_equal(ce, cg) and me == mg and int(ce.sum()) > 0
    for b in range(net.batch):
        assert util.bits_equal(de[b], dg[b]), b


@pytest.mark.skipif(not util.have_ref(), reason="reference build absent")
def test_map_mixed_sizes_equals_validate_detector_map(workdir):
    """tools/map.py's loop: batches of consecutive images whatever their sizes (heights 72..96), a partial last batch, so 7
    images at batch 2 take 4 forwards, not 7; TP / FP / FN and mAP as the reference's validate_detector_map."""
    import yolo2_light_b200 as yb
    from yolo2_light_b200 import dataset
    cfg, wts = util.model_files("tiny64", workdir)
    root = os.path.join(workdir, "mapset_tiny64_50")
    if not os.path.exists(os.path.join(root, "ref_stdout.txt")):
        util.check_map_accounting("tiny64", 0.5, workdir)
    paths, names, truth = dataset.load_validation_set(os.path.join(root, "data.cfg"))
    net = util.load(cfg, wts, 2, precision=yb.YB_PREC_FP32)

    class Counting:
        batch = net.batch
        forwards = 0

        def predict_frames_u8(self, frames, quantized=False):
            Counting.forwards += 1
            return net.predict_frames_u8(frames, quantized=quantized)

        def detect_frames(self, *a, **kw):
            return net.detect_frames(*a, **kw)

    mAP, aps, st = dataset.evaluate_map(Counting(), paths, truth, len(names), 0.5, 0.24, mixed_sizes=True)
    assert Counting.forwards == 4
    out = open(os.path.join(root, "ref_stdout.txt")).read()
    map_ref = float(re.search(r"mean average precision \(mAP\) = ([0-9.]+)", out).group(1))
    tp, fp, fn = (int(v) for v in re.search(r"TP = (\d+), FP = (\d+), FN = (\d+)", out).groups())
    assert abs(mAP - map_ref) < 5e-6
    assert (int(st["tp"]), int(st["fp"]), int(st["fn"])) == (tp, fp, fn)
