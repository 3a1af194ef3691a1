"""Tensor-core (wgmma) FP32-variant convolution: per-layer against the CPU oracle fed the GPU's own bf16 inputs,
then whole networks against the f32 oracle on the activated detection tensors (north_star: <= 1e-3 rel)."""
import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import bf16_round, tcnet
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("size,batch", [(64, 2), (96, 3), ((64, 160), 2), ((96, 32), 1)])
def test_tc_every_layer_vs_oracle_on_bf16_inputs(size, batch, workdir):
    import yolo2_light_b200 as yb
    from oracle import port
    h, w = size if isinstance(size, tuple) else (size, size)
    secs = tcnet(64)
    secs[0][1]["height"], secs[0][1]["width"] = str(h), str(w)    # non-square variants exercise H != W tiling
    net = util.load(*util.write_net(workdir, f"tcnet{h}x{w}", secs, 21), batch, precision=yb.YB_PREC_BF16_TC, fuse=0)
    x = cfgs.synthetic_images(batch, 3, h, w, seed=5)
    net.predict(x)
    kinds = util.profile_kinds(net)
    layers = net.layers
    got = [None] * net.n
    for i in range(net.n):
        got[i] = net.fetch_layer(i)
    n_tc = 0
    for i, l in enumerate(layers):
        if l["type_name"] != "CONVOLUTIONAL":
            continue
        is_tc = "conv_tc" in kinds.get(i, [])
        # the stem reads the caller's f32 NCHW image directly (tensor-core stem: rounds it to bf16 on the fly)
        xin = (bf16_round(x) if is_tc else x) if i == 0 else got[i - 1]
        n_tc += is_tc
        w = bf16_round(l["weights"]) if is_tc else l["weights"]
        exp = port.conv_fp32(xin, w, l["biases"], l["n"], l["size"], l["stride"], l["pad"], l["activation"])
        head = l["activation"] == 3
        if not head:
            exp = bf16_round(exp)
        err = util.rel_l2(got[i], exp)
        assert err <= 5e-4, (size, i, "tc" if is_tc else "simt", err)
    assert n_tc >= 14, n_tc


def s2net():
    """3x3 / stride-2 layers with 32 and 64 input channels: the parity view of k_conv_tc (one TMA box per tap), with the
    resident filter matrix (C = 32) and with streamed filter tiles over two channel blocks (C = 64), BN 64 / 128."""
    c = cfgs._conv
    return [cfgs._net(64, 64),
            c(32, 3),                   # 0 stem
            c(64, 3, 2),                # 1 C=32 s2, filters resident
            c(64, 3, 2),                # 2 C=64 s2, BN 64
            c(128, 3, 2),               # 3 C=64 s2, BN 128
            c(255, 1, bn=False, act="linear"),
            cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9)]


@pytest.mark.parametrize("hw,batch,streamed", [((64, 64), 2, 0), ((96, 160), 3, 0), ((80, 48), 5, 0), ((608, 32), 1, 0), ((96, 160), 3, 1)])
def test_tc_stride2_vs_oracle(hw, batch, streamed, workdir, monkeypatch):
    import yolo2_light_b200 as yb
    from oracle import port
    h, w = hw
    secs = s2net()
    secs[0][1]["height"], secs[0][1]["width"] = str(h), str(w)
    cfg, wts = util.write_net(workdir, f"s2net{h}x{w}", secs, 31)
    if streamed:
        monkeypatch.setenv("YB_TC_NO_BSTAT", "1")   # filter tiles streamed through the ring instead of resident (layer 1)
    net = util.load(cfg, wts, batch, precision=yb.YB_PREC_BF16_TC, fuse=0)
    x = cfgs.synthetic_images(batch, 3, h, w, seed=9)
    net.predict(x)
    layers = net.layers
    got = [net.fetch_layer(i) for i in range(net.n)]
    for i in (1, 2, 3):
        l = layers[i]
        exp = bf16_round(port.conv_fp32(got[i - 1], bf16_round(l["weights"]), l["biases"], l["n"], l["size"], l["stride"], l["pad"],
                                        l["activation"]))
        err = util.rel_l2(got[i], exp)
        assert err <= 5e-4, (hw, i, err)


def test_tc_fused_equals_unfused(workdir):
    cfg, wts = util.write_net(workdir, "tcnet64f", tcnet(64), 22)
    x = cfgs.synthetic_images(2, 3, 64, 64, seed=6)
    outs = []
    for fuse in (0, 1):
        net = util.load(cfg, wts, 2, fuse=fuse)
        net.predict(x)
        outs.append({i: o.copy() for i, o in net.detection_outputs().items()})
        launches = net.last_launches()
        outs.append(launches)
    assert outs[3] < outs[1]
    for i in outs[0]:
        assert util.rel_l2(outs[2][i], outs[0][i]) <= 2e-3, i   # residual add before vs after bf16 rounding


@pytest.mark.parametrize("name", ["tcnet", "v3_32", "spp32", "tiny64"])
def test_bf16_network_vs_f32_oracle(name, workdir):
    """Whole network, default precision, against the f32 oracle: <= 1e-3 rel-L2 on the activated yolo tensors... for
    the slim test nets the bar is 3e-3 (few channels -> less averaging of the bf16 rounding noise); the full-size
    bar is asserted in test_gpu_fullsize.py."""
    from oracle import port
    if name == "tcnet":
        cfg, wts = util.write_net(workdir, "tcnet64w", tcnet(64), 23)
        x = cfgs.synthetic_images(2, 3, 64, 64, seed=7)
    else:
        cfg, wts = util.model_files(name, workdir)
        x = util.images(name, 2)
    net = util.load(cfg, wts, 2)
    net.predict(x)
    layers = net.layers
    exp = [port.run_network(layers, x[b:b + 1]) for b in range(2)]
    for i, o in net.detection_outputs().items():
        e = np.concatenate([exp[b][i] for b in range(2)], 0).reshape(o.shape)
        err = util.rel_l2(o, e)
        assert err <= 3e-3, (name, i, err)


def deepknet(h, w):
    """Deep-K layers on small grids: every tensor-core layer has far fewer tiles than the GPU has SMs, so each CTA
    runs at most a few long work items."""
    c = cfgs._conv
    return [cfgs._net(w, h),
            c(32, 3),                   # 0 stem
            c(256, 3, 2),               # 1 s2, K = 9*32
            c(256, 3),                  # 2 K = 9*256: 36 K-blocks
            c(128, 1),                  # 3 1x1, K = 256
            c(256, 3),                  # 4 + fused shortcut, K = 9*128
            ("shortcut", {"from": "-3", "activation": "linear"}),   # 5
            c(512, 3),                  # 6 several filter tiles
            c(128, 3),                  # 7 K = 9*512: resident-B not possible, filter tiles streamed
            c(64, 3),                   # 8 K = 9*128
            c(255, 1, bn=False, act="linear"),   # 9 head (fused yolo), K = 64
            cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9),
            ("route", {"layers": "-4"}),                                # 11 -> layer 7
            c(255, 3, bn=False, act="linear"),   # 12 f32 head with deep K (9*128), generic epilogue
            cfgs._yolo("3,4,5", cfgs.COCO_ANCHORS, 9)]


@pytest.mark.parametrize("fuse", [0, 1])
@pytest.mark.parametrize("h,w,batch", [(32, 32, 2), (64, 32, 3), (96, 96, 4)])
def test_tc_deepknet_vs_f32_oracle(h, w, batch, fuse, workdir):
    """The deep-K network against the f32 oracle on the detection tensors, with the bar of the other slim nets (see
    test_bf16_network_vs_f32_oracle), fused and unfused, after repeated launches of the same engine."""
    from oracle import port
    cfg, wts = util.write_net(workdir, f"deepk{h}x{w}", deepknet(h, w), 31)
    x = cfgs.synthetic_images(batch, 3, h, w, seed=9)
    net = util.load(cfg, wts, batch, fuse=fuse)
    for rep in range(3):
        net.predict(x)
    assert net.get_info("tc_layers") >= 9
    layers = net.layers
    exp = [port.run_network(layers, x[b:b + 1]) for b in range(batch)]
    for i, o in net.detection_outputs().items():
        e = np.concatenate([exp[b][i] for b in range(batch)], 0).reshape(o.shape)
        err = util.rel_l2(o, e)
        assert err <= 3e-3, (h, w, batch, fuse, i, err)


@pytest.mark.parametrize("name,q", [("tiny64", 1), ("xnor64", 0), ("tiny_w96_h64", 1)])
def test_tf32_heads_of_exact_networks(name, q, workdir):
    """The float detection heads of the INT8 / XNOR networks run on the tf32 wgmma in the default precision (their
    result feeds no integer layer); everything upstream stays bit-exact, the detections stay within the FP32 bar of
    the all-f32 engine (north_star: <= 1e-3 rel)."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files(name, workdir)
    B = 3
    x = util.images(name, B)
    fast = util.load(cfg, wts, B, quantized=q)
    fast.predict(x, quantized=bool(q))
    kinds = [k for _, k, _ in fast.profile(quantized=bool(q))]
    assert "conv_tc_tf32" in kinds, kinds
    exact = util.load(cfg, wts, B, quantized=q, precision=yb.YB_PREC_FP32)
    exact.predict(x, quantized=bool(q))
    assert "conv_tc_tf32" not in [k for _, k, _ in exact.profile(quantized=bool(q))]
    for i, o in fast.detection_outputs().items():
        err = util.rel_l2(o, exact.detection_outputs()[i])
        assert err <= 1e-3, (name, i, err)
    # the integer layers did not notice: raw accumulators / counts of the last integer layer are identical
    fast.set_option("keep_counts", 1); exact.set_option("keep_counts", 1)
    fast.predict(x, quantized=bool(q)); exact.predict(x, quantized=bool(q))
    ints = [i for i, l in enumerate(fast.layers) if l["type_name"] == "CONVOLUTIONAL" and (l["xnor"] or (q and i >= 1 and l["activation"] != 3))]
    a = fast.fetch_counts(ints[-1], quantized=bool(q)); b = exact.fetch_counts(ints[-1], quantized=bool(q))
    assert a is not None and np.array_equal(a, b)
