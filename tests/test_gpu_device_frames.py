"""Frames already in device memory (yb_network_predict_device_frames, yb_network_submit_device_frames): RGB, BGR, planar
RGB and NV12 frames, made with torch, in padded, odd-offset and tightly sized layouts.  Each must give bit for bit what
its equivalent host frame gives through the host calls: the resized input, the detection tensors, the rows and the
counts.  The calls are ordered with the caller's stream, and memory that is not the network device's is rejected."""
import numpy as np
import pytest

import ybtest_util as util
from device_frames_util import GOLDEN_NV12, LAYOUTS, device_frame, equivalent_host_frame, random_frame
from ybtest_util import INPUT_SETS, mixed_net

pytestmark = pytest.mark.gpu

FORMATS = ["rgb", "bgr", "planar", "nv12"]
# NV12 needs even sizes: the sets of test_gpu_frames without the 1-pixel and odd sizes, sizes rounded up to even
NV12_SETS = [[(2, 40), (50, 2), (64, 64), (34, 18)],
             [(200, 198), (98, 132), (4500, 6)],
             [(8, 10)]]


def _sets(fmt):
    return NV12_SETS if fmt == "nv12" else INPUT_SETS


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    import yolo2_light_b200 as yb
    net = util.load(*util.model_files("tiny64", str(tmp_path_factory.mktemp("device_frames"))), 4, precision=yb.YB_PREC_FP32)
    return net


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("k", range(3))
@pytest.mark.parametrize("fmt", FORMATS)
def test_resized_input_equals_host_path(tiny, fmt, k, layout):
    rng = np.random.default_rng(300 + 7 * k + FORMATS.index(fmt))
    frames = [random_frame(fmt, w, h, rng) for w, h in _sets(fmt)[k]]
    tiny.predict_frames_u8([equivalent_host_frame(fmt, f) for f in frames])
    exp = tiny.fetch_input().copy()
    dev = [device_frame(fmt, f, layout, nv12_pair=(fmt == "nv12" and layout == "padded")) for f in frames]
    tiny.predict_device_frames(dev, fmt=fmt)
    got = tiny.fetch_input()
    for b in range(len(frames)):
        assert util.bits_equal(got[b], exp[b]), (fmt, k, layout, b, frames[b].shape)
    tail = got[len(frames):]
    assert tail.size == 0 or not tail.view(np.uint32).any()


def test_nv12_equals_cv2_through_the_host_path(tiny):
    g = np.load(GOLDEN_NV12)
    n = len([f for f in g.files if f.startswith("nv12_")])
    for i in range(n):
        for layout in LAYOUTS:
            tiny.predict_frames_u8([g[f"rgb_{i}"]])
            exp = tiny.fetch_input()[0].copy()
            tiny.predict_device_frames([device_frame("nv12", g[f"nv12_{i}"], layout)], fmt="nv12")
            assert util.bits_equal(tiny.fetch_input()[0], exp), (i, layout)
            tiny.predict_frames_u8([g[f"bgr_{i}"][..., ::-1].copy()])
            assert util.bits_equal(tiny.fetch_input()[0], exp), (i, "bgr")


# mixed sizes (the network size among them) and a partial batch; all even, so that NV12 takes them too
DET_BATCHES = [[(120, 96), (64, 64), (32, 200)], [(300, 170)], [(64, 64), (2, 2)], [(64, 64)] * 2]


@pytest.mark.parametrize("kind", ["tiny64_fp32", "tiny64_bf16", "s2chain", "tiny64_q1", "xnor64"])
def test_detections_equal_host_frames(kind, workdir):
    net, q = mixed_net(kind, workdir)
    rng = np.random.default_rng(17)
    total = 0
    for fmt in FORMATS:
        for letter in (0, 1):
            for sizes in DET_BATCHES:
                frames = [random_frame(fmt, w, h, rng) for w, h in sizes]
                t = net.submit_frames_u8([equivalent_host_frame(fmt, f) for f in frames], 0.3, 0.45, relative=0,
                                         letter=letter, max_rows=2048, quantized=q)
                de, ce, _ = net.collect_detections(t, quantized=q)
                dev = [device_frame(fmt, f, "odd_offset") for f in frames]
                t = net.submit_device_frames(dev, 0.3, fmt=fmt, relative=0, letter=letter, max_rows=2048, quantized=q)
                dg, cg, _ = net.collect_detections(t, quantized=q)
                assert len(dg) == len(sizes) and np.array_equal(ce, cg), (kind, fmt, letter, sizes, ce, cg)
                for b in range(len(sizes)):
                    assert util.bits_equal(de[b], dg[b]), (kind, fmt, letter, sizes, b)
                total += int(ce.sum())
                # the synchronous call makes the same detection tensors
                net.predict_frames_u8([equivalent_host_frame(fmt, f) for f in frames], quantized=q)
                he = {i: o.copy() for i, o in net.detection_outputs().items()}
                net.predict_device_frames(dev, fmt=fmt, quantized=q)
                for i, o in net.detection_outputs().items():
                    assert util.bits_equal(o, he[i]), (kind, fmt, sizes, i)
    assert total > 0


def test_stream_ordering_with_the_producer(workdir):
    """The producer stream sleeps, writes the frames, submits them without synchronising and then overwrites them: the
    engine reads what was written before the call.  Device and host submits share the three slots of one network."""
    import torch
    net, q = mixed_net("s2chain", workdir)
    rng = np.random.default_rng(23)
    sizes = [(120, 96), (64, 64), (32, 200)]
    plan = ["rgb", "host", "nv12", "bgr", "host", "planar", "nv12"]
    contents = [[random_frame("rgb" if f == "host" else f, w, h, rng) for w, h in sizes] for f in plan]
    expected = []
    for f, fr in zip(plan, contents):
        t = net.submit_frames_u8([equivalent_host_frame("rgb" if f == "host" else f, x) for x in fr], 0.3, 0.45,
                                 relative=0, max_rows=2048, quantized=q)
        expected.append(net.collect_detections(t, quantized=q)[:2])
    assert sum(int(c.sum()) for _, c in expected) > 0
    s = torch.cuda.Stream()
    # one set of device frames per format, rewritten for every batch of that format; the sources of the writes stay
    # allocated until the end, so that no allocation of this test reuses their memory while the stream still reads them
    bufs = {f: [device_frame(f, np.zeros_like(x), "padded") for x in fr] for f, fr in zip(plan, contents) if f != "host"}
    new = [[torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in fr] for fr in contents]
    junk = [[torch.from_numpy(255 - np.ascontiguousarray(x)).cuda() for x in fr] for fr in contents]
    torch.cuda.synchronize()
    inflight, got = [], []
    for k, (f, fr) in enumerate(zip(plan, contents)):
        if len(inflight) == 3:
            got.append(net.collect_detections(inflight.pop(0), quantized=q)[:2])
        if f == "host":
            inflight.append(net.submit_frames_u8(fr, 0.3, 0.45, relative=0, max_rows=2048, quantized=q))
            continue
        with torch.cuda.stream(s):
            torch.cuda._sleep(20_000_000)                 # the writes and the engine's reads would race without the hand-off
            for d, x in zip(bufs[f], new[k]):
                d.copy_(x)
            inflight.append(net.submit_device_frames(bufs[f], 0.3, fmt=f, relative=0, max_rows=2048, quantized=q,
                                                     stream=s.cuda_stream))
            for d, x in zip(bufs[f], junk[k]):            # the next producer write, right after the call
                d.copy_(x)
    while inflight:
        got.append(net.collect_detections(inflight.pop(0), quantized=q)[:2])
    torch.cuda.synchronize()
    for k, ((de, ce), (dg, cg)) in enumerate(zip(expected, got)):
        assert np.array_equal(ce, cg), (k, plan[k], ce, cg)
        for b in range(len(de)):
            assert util.bits_equal(de[b], dg[b]), (k, plan[k], b)


class _Cai:
    def __init__(self, ptr, shape, strides):
        self.__cuda_array_interface__ = {"shape": shape, "strides": strides, "typestr": "|u1", "data": (ptr, False),
                                         "version": 3}


def test_host_and_pinned_memory_are_rejected(tiny):
    import torch
    import yolo2_light_b200 as yb
    host = np.zeros((8, 8, 3), np.uint8)
    pinned = torch.zeros((8, 8, 3), dtype=torch.uint8).pin_memory()
    for obj, kind in ((_Cai(host.ctypes.data, (8, 8, 3), None), "host memory"),
                      (_Cai(pinned.data_ptr(), (8, 8, 3), None), "pinned host memory")):
        with pytest.raises(yb.YbError, match=f"predict_device_frames: frame 0 is {kind}, not device memory of device 0"):
            tiny.predict_device_frames([obj])
        with pytest.raises(yb.YbError, match=f"submit_device_frames: frame 0 is {kind}, not device memory of device 0"):
            tiny.submit_device_frames([obj], 0.5)
    # NV12: the chroma plane is checked too
    y = torch.zeros((8, 8), dtype=torch.uint8, device="cuda")
    with pytest.raises(yb.YbError, match="frame 0 chroma is pinned host memory"):
        tiny.predict_device_frames([(y, _Cai(pinned.data_ptr(), (4, 8), None))], fmt="nv12")
    # the network still serves device frames afterwards
    tiny.predict_device_frames([torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda")])


def test_other_device_memory_is_rejected(tiny):
    import torch
    import yolo2_light_b200 as yb
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    other = torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda:1")
    with pytest.raises(yb.YbError, match="frame 0 is device memory of device 1, not device memory of device 0"):
        tiny.predict_device_frames([other])
