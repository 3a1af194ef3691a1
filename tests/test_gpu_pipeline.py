"""The three-slot pipeline one network shares between raw-tensor tickets (yb_network_submit / yb_network_collect) and
detection tickets (yb_network_submit_u8, yb_network_submit_frames_u8 and yb_network_submit_device_frames, collected with
yb_network_collect_detections): both kinds interleaved on every slot, a full pipeline, tickets collected with the wrong
call, and a network freed with tickets still in flight.  Every result is compared bitwise with the synchronous calls on the
same inputs."""
import gc

import numpy as np
import pytest

import ybtest_util as util
from device_frames_util import device_frame, equivalent_host_frame, random_frame
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu

B, W, H = 3, 160, 128
DEPTH = 3                      # batches in flight
THRESH, NMS, MAX_ROWS = 0.3, 0.45, 2048
KINDS = ("raw", "u8", "frames", "device")


def _job(net, kind, seed, q):
    """One batch of `kind` and what the synchronous calls make of it: the detection tensors for "raw", else (rows per
    image, counts)."""
    rng = np.random.default_rng(seed)
    job = {"kind": kind}
    if kind == "raw":
        job["x"] = cfgs.synthetic_images(B, 3, H, W, seed=seed)
        net.predict(job["x"], quantized=q)
        job["exp"] = {i: o.copy() for i, o in net.detection_outputs().items()}
        return job
    if kind == "u8":   # a whole batch of frames of the network size: the stem reads them where it can
        job["f"] = rng.integers(0, 256, size=(B, H, W, 3), dtype=np.uint8)
        net.predict_image_u8(job["f"], quantized=q)
        dets, counts = net.detect(W, H, THRESH, NMS, max_rows=MAX_ROWS, quantized=q)
    else:              # a partial batch of frames of their own sizes, from the host or as NV12 in device memory
        sizes = [(120, 96), (W, H)] if kind == "frames" else [(64, 64), (W, H), (200, 150)]
        fmt = "rgb" if kind == "frames" else "nv12"
        frames = [random_frame(fmt, w, h, rng) for w, h in sizes]
        job["frames"] = [equivalent_host_frame(fmt, f) for f in frames]
        if kind == "device":
            job["dev"] = [device_frame(fmt, f, "padded") for f in frames]
        net.predict_frames_u8(job["frames"], quantized=q)
        dets, counts = net.detect_frames(sizes, THRESH, NMS, max_rows=MAX_ROWS, quantized=q)
    job["exp"] = ([d.copy() for d in dets], counts.copy())
    return job


def _submit(net, job, q):
    kind = job["kind"]
    if kind == "raw":
        return net.submit(job["x"], quantized=q)
    if kind == "u8":
        return net.submit_u8(job["f"], THRESH, NMS, max_rows=MAX_ROWS, quantized=q)
    if kind == "frames":
        return net.submit_frames_u8(job["frames"], THRESH, NMS, max_rows=MAX_ROWS, quantized=q)
    return net.submit_device_frames(job["dev"], THRESH, fmt="nv12", nms=NMS, max_rows=MAX_ROWS, quantized=q)


def _collect_and_check(net, job, ticket, q, what):
    """Collects the ticket with the call of its kind and compares with the synchronous results; returns the candidates."""
    if job["kind"] == "raw":
        got = net.collect(ticket, quantized=q)
        assert set(got) == set(job["exp"]), what
        for i, o in got.items():
            assert util.bits_equal(o, job["exp"][i]), (what, i)
        return 0
    dets, counts, moved = net.collect_detections(ticket, quantized=q)
    de, ce = job["exp"]
    assert np.array_equal(counts, ce), (what, counts, ce)
    assert len(dets) == len(de), what
    for b in range(len(de)):
        assert util.bits_equal(dets[b], de[b]), (what, b)
    # exactly the candidate rows and the counts of the whole batch cross PCIe
    assert moved == sum(d.nbytes for d in dets) + B * 4, what
    return int(counts.sum())


@pytest.mark.parametrize("q", [0, 1])
def test_raw_and_detection_tickets_interleave_on_every_slot(q, workdir):
    net = util.load(*util.write_net(workdir, "pipe_tiny", cfgs.slim(cfgs.yolov3_tiny, 2, W, H), 23), B, quantized=q)
    # 16 batches cycling through the four kinds over three slots: every slot serves every kind, both after a ticket of
    # the same mode and after one of the other mode
    jobs = [_job(net, KINDS[k % len(KINDS)], 100 + k, bool(q)) for k in range(16)]
    inflight, candidates = [], 0
    for k, job in enumerate(jobs):
        if len(inflight) == DEPTH:
            j, t = inflight.pop(0)
            candidates += _collect_and_check(net, jobs[j], t, bool(q), j)
        inflight.append((k, _submit(net, job, bool(q))))
    while inflight:
        j, t = inflight.pop(0)
        candidates += _collect_and_check(net, jobs[j], t, bool(q), j)
    assert candidates > 20


def test_full_pipeline_refuses_and_runs_on(workdir):
    import yolo2_light_b200 as yb
    net = util.load(*util.write_net(workdir, "pipe_tiny", cfgs.slim(cfgs.yolov3_tiny, 2, W, H), 23), B)
    jobs = [_job(net, KINDS[k % len(KINDS)], 200 + k, False) for k in range(7)]
    inflight = [(k, _submit(net, jobs[k], False)) for k in range(DEPTH)]
    for k in (DEPTH, DEPTH + 1):    # a fourth batch: device frames, then raw
        with pytest.raises(yb.YbError, match="pipeline full"):
            _submit(net, jobs[k], False)
    j, t = inflight.pop(0)
    _collect_and_check(net, jobs[j], t, False, j)
    # a submit refused for its arguments takes no slot: the next one takes the slot that was freed
    with pytest.raises(yb.YbError, match="max_rows"):
        net.submit_u8(jobs[1]["f"], THRESH, NMS, max_rows=0)
    for k in range(DEPTH, len(jobs)):
        inflight.append((k, _submit(net, jobs[k], False)))
        j, t = inflight.pop(0)
        _collect_and_check(net, jobs[j], t, False, j)
    for j, t in inflight:
        _collect_and_check(net, jobs[j], t, False, j)


def test_ticket_collected_with_the_wrong_call(workdir):
    import yolo2_light_b200 as yb
    net = util.load(*util.write_net(workdir, "pipe_tiny", cfgs.slim(cfgs.yolov3_tiny, 2, W, H), 23), B)
    raw, det = _job(net, "raw", 300, False), _job(net, "frames", 301, False)
    t_raw, t_det = _submit(net, raw, False), _submit(net, det, False)
    with pytest.raises(yb.YbError, match="collect_detections: bad ticket"):
        net.collect_detections(t_raw)
    with pytest.raises(yb.YbError, match="collect: bad ticket"):
        net.collect(t_det)
    _collect_and_check(net, raw, t_raw, False, "raw")
    _collect_and_check(net, det, t_det, False, "det")


def test_network_freed_with_tickets_in_flight(workdir):
    cfg, wts = util.write_net(workdir, "pipe_v3", cfgs.slim(cfgs.yolov3, 4, W, H), 23)
    net = util.load(cfg, wts, B)
    jobs = [_job(net, kind, 400 + k, False) for k, kind in enumerate(("raw", "u8", "device"))]
    for job in jobs:
        _submit(net, job, False)
    del net     # three uncollected tickets, of both kinds
    gc.collect()
    fresh = util.load(cfg, wts, B)
    tickets = [_submit(fresh, job, False) for job in jobs]
    for k, (job, t) in enumerate(zip(jobs, tickets)):
        _collect_and_check(fresh, job, t, False, k)
