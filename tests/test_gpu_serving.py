"""The serving-side entry points added around the hot path, all through the C ABI:
  * yb_network_submit_u8 / yb_network_collect_detections (u8 frames -> device resize -> forward -> device decode + NMS, three
    batches in flight) against the synchronous calls on the same frames;
  * yb_network_predict_batch (several engine replicas in ONE process, weights broadcast once) against the one-GPU predict,
    from Python and from a plain-C host program (tests/c/batch_multi_gpu.c);
  * forward_convolutional_layer_b200[_q](layer l, network_state state) and network_predict_b200_batch of the reference-side
    glue, behind the reference's UNMODIFIED host code (oracle/_ref/libyolo2ref_dropin.so)."""
import os
import subprocess

import numpy as np
import pytest

import ybtest_util as util
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu
ROOT = util.ROOT


@pytest.mark.parametrize("builder,slim,q,thresh,fw,fh", [(cfgs.yolov3_tiny, 2, 0, 0.3, 120, 96), (cfgs.yolov3, 4, 0, 0.3, 120, 96),
                                                        (cfgs.yolov3_tiny, 2, 1, 0.3, 120, 96), (cfgs.tiny_yolo_obj_xnor, 2, 0, 0.05, 120, 96),
                                                        # frames of exactly the network size: the stem reads the 8-bit frames itself
                                                        (cfgs.yolov3, 4, 0, 0.3, 160, 128), (cfgs.yolov3_tiny, 2, 0, 0.3, 160, 128)])
def test_pipelined_u8_detections_equal_sync_calls(builder, slim, q, thresh, fw, fh, workdir):
    B, W, H = 3, 160, 128
    net = util.load(*util.write_net(workdir, f"srv_{builder.__name__}_{q}", cfgs.slim(builder, slim, W, H), 51), B, quantized=q)
    rng = np.random.default_rng(5)
    frames = [rng.integers(0, 256, size=(B, fh, fw, 3), dtype=np.uint8) for _ in range(5)]   # 120x96 frames are resized on the device
    # expected: the synchronous pair predict_image_u8 + detect, frame set by frame set
    exp = []
    for f in frames:
        net.predict_image_u8(f, quantized=bool(q))
        dets, counts = net.detect(fw, fh, thresh, 0.45, max_rows=2048, quantized=bool(q))
        exp.append(([d.copy() for d in dets], counts.copy()))
    assert sum(int(c.sum()) for _, c in exp) > 20
    inflight, got, moved = [], [], 0
    for f in frames:
        if len(inflight) == 3:
            d, c, m = net.collect_detections(inflight.pop(0), quantized=bool(q))
            got.append((d, c)); moved += m
        inflight.append(net.submit_u8(f, thresh, 0.45, max_rows=2048, quantized=bool(q)))
    while inflight:
        d, c, m = net.collect_detections(inflight.pop(0), quantized=bool(q))
        got.append((d, c)); moved += m
    for k, ((de, ce), (dg, cg)) in enumerate(zip(exp, got)):
        assert np.array_equal(ce, cg), (k, ce, cg)
        for b in range(B):
            assert util.bits_equal(de[b], dg[b]), (k, b)
    rowbytes = sum(d.nbytes for de, _ in exp for d in de)
    assert moved == rowbytes + len(frames) * B * 4      # exactly the candidate rows + the counts cross PCIe


def test_predict_batch_two_replicas_equals_single_gpu(workdir):
    import torch
    B, W, H = 2, 96, 96
    net = util.load(*util.write_net(workdir, "srv_pb_v3", cfgs.slim(cfgs.yolov3, 4, W, H), 51), B)
    nimg = 3 * 2 * B + 1      # three rounds over two replicas and a partial last shard
    x = cfgs.synthetic_images(nimg, 3, H, W, seed=77)
    exp = {}
    for first in range(0, nimg, B):
        xb = np.zeros((B, 3, H, W), np.float32)
        cnt = min(B, nimg - first)
        xb[:cnt] = x[first:first + cnt]
        net.predict(xb)
        for i, o in net.detection_outputs().items():
            exp.setdefault(i, np.zeros((nimg,) + o.shape[1:], np.float32))[first:first + cnt] = o[:cnt]
    two = torch.cuda.device_count() >= 2
    net.set_devices([0, 1] if two else [0, 0])
    got = net.predict_batch(x, 2)
    assert net.replication() in (("nccl", "peer-copy") if two else ("peer-copy",))
    for i, e in exp.items():
        assert util.bits_equal(got[i].reshape(e.shape), e), i
    # one replica through the same call
    net.set_devices([0])
    got1 = net.predict_batch(x, 1)
    for i, e in exp.items():
        assert util.bits_equal(got1[i].reshape(e.shape), e), i


@pytest.mark.parametrize("builder,slim,q", [(cfgs.yolov3_tiny, 2, 0), (cfgs.yolov3_tiny, 2, 1), (cfgs.tiny_yolo_obj_xnor, 2, 0)])
def test_c_host_program_drives_two_replicas(builder, slim, q, workdir):
    """tests/c/batch_multi_gpu.c: plain C, links only libyolo2_light_b200.so."""
    exe = os.path.join(workdir, "batch_multi_gpu")
    if not os.path.exists(exe):
        subprocess.check_call(["gcc", "-O1", "-std=c99", "-Wall", "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "c", "batch_multi_gpu.c"), "-o", exe,
                               "-L", os.path.join(ROOT, "yolo2_light_b200"), "-lyolo2_light_b200",
                               "-Wl,-rpath," + os.path.join(ROOT, "yolo2_light_b200")])
    cfg, wts = util.write_net(workdir, f"srv_c_{builder.__name__}_{q}", cfgs.slim(builder, slim, 96, 64), 51)
    r = subprocess.run([exe, cfg, wts, "2", "9", str(q)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "bit-identical" in r.stdout


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libyolo2ref_dropin.so")), reason="drop-in library not built")
@pytest.mark.parametrize("name,q", [("tiny64", 1), ("xnor64", 0), ("tiny64", 0)])
def test_forward_convolutional_layer_b200_slot(name, q, workdir):
    """forward_convolutional_layer_b200[_q](layer l, network_state state): the reference's by-value per-layer call shape, with
    the reference's own layer loop around it (every other layer type runs the reference's CPU code)."""
    from oracle import ref
    cfg, wts = util.model_files(name, workdir)
    rnet = ref.RefNet(cfg, wts, 1, q, 7, kind="dropin")
    x = util.images(name, 1)
    rnet.predict(x)                                            # reference CPU path: every layer's l.output
    expected = [rnet.output(i).copy() for i in range(rnet.n)]
    n_int = n_f = 0
    for i, L in enumerate(rnet.layers):
        if L["type_name"] != "CONVOLUTIONAL":
            continue
        xin = x if i == 0 else expected[i - 1]
        got = rnet.forward_conv_b200(i, xin, use_q_rule=bool(q)).copy()
        integer = L["xnor"] or (q and i >= 1 and L["activation_name"] != "LINEAR")
        if integer:      # XNOR popcount / INT8 accumulators + the reference's float epilogue: bit-exact
            assert util.bits_equal(got, expected[i]), (name, q, i, float(np.abs(got - expected[i]).max()))
            n_int += 1
        else:            # FP32 variant on bf16 tensor cores
            assert util.rel_l2(got, expected[i]) <= 1e-2, (name, q, i)
            n_f += 1
    assert n_f >= 1 and (n_int >= 5 or (name == "tiny64" and q == 0))


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libyolo2ref_dropin.so")), reason="drop-in library not built")
def test_dropin_predict_batch_behind_reference_host_code(workdir):
    from oracle import ref
    cfg, wts = util.model_files("tiny64", workdir)
    rnet = ref.RefNet(cfg, wts, 1, 0, 7, kind="dropin")
    x = util.images("tiny64", 5)
    got = rnet.predict_b200_batch(x, 1)
    for b in range(5):
        e = rnet.predict_b200(x[b:b + 1]).reshape(-1)
        assert util.bits_equal(got[b], e), b
