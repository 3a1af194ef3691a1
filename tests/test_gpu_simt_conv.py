"""The CUDA-core implicit-GEMM convolution (k_conv_simt) on the layers only it takes: INT8 layers the s8 wgmma tile refuses, XNOR
layers off the s8 wgmma with more than 2 sign words per tap, and bf16 layers the tensor cores refuse.  Each network's op list
shows the path runs; the results are checked against the CPU oracle.  GPU box only."""
import numpy as np
import pytest

import ybtest_util as util
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu

B = 2


def test_int8_layers_outside_the_tensor_core_tile(workdir):
    """3x3 / stride 2 on 13 x 13 (odd: 13 -> 7), 1x1 / stride 2, and 4 filters: s32 accumulators and outputs bit-exact, per layer
    and over the whole network"""
    from oracle import port
    c = cfgs._conv
    secs = [cfgs._net(26, 26, [16] * 8), c(16, 3), ("maxpool", {"size": "2", "stride": "2"}),
            c(32, 3, 2),     # 2: 13 -> 7
            c(32, 1, 2),     # 3: 1x1 / 2, 7 -> 4
            c(4, 3),         # 4: 4 filters
            c(18, 1, bn=False, act="linear")]
    net = util.load(*util.write_net(workdir, "simt_int8", secs, 41), B, quantized=1, fuse=0, keep_counts=True)
    x = cfgs.synthetic_images(B, 3, 26, 26, seed=42)
    net.predict(x, quantized=True)
    kinds = util.profile_kinds(net, True)
    for i in (2, 3, 4):
        assert "conv_int8" in kinds[i], (i, kinds[i])
    outs = util.oracle_outs(net, x, 1)
    for i in (2, 3, 4):
        l = net.layer(i)
        args = (l["weights_int8"], l["biases"], l["input_quant_multipler"], l["weights_quant_multipler"], l["n"], l["size"],
                l["stride"], l["pad"], l["activation"])
        got = net.forward_convolutional_layer(i, outs[i - 1], variant=1)
        assert util.bits_equal(got, port.conv_int8(outs[i - 1], *args)), i
        _, acc = port.conv_int8(outs[i - 1], *args, want_acc=True)
        assert np.array_equal(net.fetch_counts(i, quantized=True), acc), i
        out = net.fetch_layer(i, quantized=True)
        assert util.bits_equal(out, outs[i].reshape(out.shape)), i


def test_xnor_layers_on_the_general_popcount_kernel(workdir):
    """3x3 / 1 / 1 XNOR layers with C = 72 (3 sign words, not a multiple of 16) and with C = 96 but 4 filters: popcounts and
    outputs bit-exact"""
    from oracle import port
    c = cfgs._conv
    xn = {"xnor": 1, "bin_output": 1}
    secs = [cfgs._net(20, 20), c(72, 3),
            c(96, 3, **xn),  # 1: C = 72
            c(4, 3, **xn),   # 2: C = 96, 4 filters
            c(18, 1, bn=False, act="linear")]
    net = util.load(*util.write_net(workdir, "simt_xnor", secs, 43), B, fuse=0, keep_counts=True)
    x = cfgs.synthetic_images(B, 3, 20, 20, seed=44)
    net.predict(x)
    kinds = util.profile_kinds(net)
    for i in (1, 2):
        assert "conv_xnor" in kinds[i], (i, kinds[i])
    outs = util.oracle_outs(net, x, 0)
    for i in (1, 2):
        l = net.layer(i)
        exp, cnt = port.conv_xnor(outs[i - 1], l["weights"], l["biases"], l["mean_arr"], l["n"], l["size"], l["activation"],
                                  want_counts=True)
        got = net.forward_convolutional_layer(i, outs[i - 1], variant=0)
        assert util.bits_equal(got, exp), i
        assert np.array_equal(net.fetch_counts(i), cnt), i
        out = net.fetch_layer(i)
        assert util.bits_equal(out, outs[i].reshape(out.shape)), i


def test_bf16_layer_the_tensor_cores_refuse(workdir):
    """3x3 / stride 2 on 13 x 13 in a bf16 network runs on CUDA cores, between tensor-core layers"""
    import yolo2_light_b200 as yb
    from oracle import port
    c = cfgs._conv
    secs = [cfgs._net(26, 26), c(16, 3), ("maxpool", {"size": "2", "stride": "2"}),
            c(32, 3, 2),     # 2: 13 -> 7
            c(32, 3),        # 3
            c(255, 1, bn=False, act="linear"), cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9)]
    net = util.load(*util.write_net(workdir, "simt_bf16", secs, 45), B, precision=yb.YB_PREC_BF16_TC, fuse=0)
    x = cfgs.synthetic_images(B, 3, 26, 26, seed=46)
    net.predict(x)
    kinds = util.profile_kinds(net)
    assert "conv_simt" in kinds[2] and "conv_tc" in kinds[3], kinds
    l = net.layer(2)
    exp = util.bf16_round(port.conv_fp32(net.fetch_layer(1), l["weights"], l["biases"], l["n"], l["size"], l["stride"], l["pad"],
                                    l["activation"]))
    err = util.rel_l2(net.fetch_layer(2), exp)
    assert err <= 5e-4, err
