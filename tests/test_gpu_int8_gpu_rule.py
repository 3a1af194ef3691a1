"""The GPU build's INT8 mode (YB_QUANT_GPU = 2, network_predict_gpu_cudnn_quantized) on the H100: the INT8 layers are the
parser's l.quantized, with the saturating input conversion and the unscaled epilogue; everything else as in the float forward
with f32 activations.  Checked bit for bit against the oracle's forward under the GPU rule (tests/rule_oracle.py) at YB_PREC_FP32, and against the
oracle's INT8 convolution on the engine's own inputs at the default precision, where the float layers run on tf32.  GPU box only."""
import numpy as np
import pytest

import rule_oracle as ro
import ybtest_util as util
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu
Q = 2


def _int8_layers(net):
    return [i for i, l in enumerate(net.layers) if l["type_name"] == "CONVOLUTIONAL" and l["quantized"]]


def _assert_bit_exact(net, outs, need=()):
    got = util.fetch_all(net, Q)
    for i in need:
        assert i in got, i
    for i, o in got.items():
        assert util.bits_equal(o, np.asarray(outs[i]).reshape(o.shape)), i
    for i, o in net.detection_outputs().items():
        assert util.bits_equal(o, np.asarray(outs[i]).reshape(o.shape)), i
    return got


@pytest.fixture(scope="module")
def tiny416(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("tiny416"))
    cfg, wts = util.write_net(d, "tiny416", cfgs.yolov3_tiny(416, 416), 41)
    x = cfgs.synthetic_images(4, 3, 416, 416, seed=42)
    return cfg, wts, x


def test_yolov3_tiny_416_fp32_bit_exact(tiny416):
    """yolov3-tiny 416, batch 4, YB_PREC_FP32: the s32 accumulators of every INT8 layer, every layer's output and the yolo
    tensors are those of the oracle's forward_network_gpu_cudnn_quantized loop."""
    import yolo2_light_b200 as yb
    from oracle import port
    cfg, wts, x = tiny416
    net = util.load(cfg, wts, 4, quantized=1, precision=yb.YB_PREC_FP32, fuse=0, keep_counts=True)
    assert _int8_layers(net) == [2, 4, 6, 8, 10, 12]
    net.predict(x, quantized=Q)
    layers = net.layers
    outs = ro.forward(layers, x, Q)
    for i in _int8_layers(net):
        _, acc = util.oracle_layer(layers[i], i, outs[i - 1], Q)
        assert np.array_equal(net.fetch_counts(i, quantized=Q), acc), i
    got = _assert_bit_exact(net, outs)
    assert len(got) >= 20
    # the CPU rule is a different computation on the same network
    cpu = port.run_network(layers, x, quantized=True)
    assert not util.bits_equal(cpu[23], outs[23])


def test_yolov3_tiny_416_default_precision(tiny416):
    """Default precision: each INT8 layer is bit-exact against the oracle's INT8 convolution of the engine's own input; every
    float convolution but the 3-channel stem runs on tf32; the yolo tensors stay within rel-L2 1e-3 of YB_PREC_FP32."""
    import yolo2_light_b200 as yb
    cfg, wts, x = tiny416
    net = util.load(cfg, wts, 4, quantized=1, fuse=0)
    net.predict(x, quantized=Q)
    layers = net.layers
    for i in _int8_layers(net):
        exp, _ = util.oracle_layer(layers[i], i, net.fetch_layer(i - 1, quantized=Q), Q)
        assert util.bits_equal(net.fetch_layer(i, quantized=Q), exp), i
        assert net.tc_plan(i, quantized=Q)["kind"] == "s8_gpu", i
    floats = [i for i, l in enumerate(layers) if l["type_name"] == "CONVOLUTIONAL" and not l["quantized"] and i > 0]
    assert floats == [13, 14, 15, 18, 21, 22]
    for i in floats:
        assert net.tc_plan(i, quantized=Q)["kind"] == "tf32", i
    fused = util.load(cfg, wts, 4, quantized=1)            # the production engine: every fusion on
    fused.predict(x, quantized=Q)
    exact = util.load(cfg, wts, 4, quantized=1, precision=yb.YB_PREC_FP32)
    exact.predict(x, quantized=Q)
    ref = exact.detection_outputs()
    for i, o in fused.detection_outputs().items():
        err = util.rel_l2(o, ref[i])
        assert err <= 1e-3, (i, err)
    # the production engine runs the tensor-core plans of the GPU rule
    assert fused.tc_plan(15, quantized=Q)["kind"] == "tf32" and fused.tc_plan(4, quantized=Q)["kind"] == "s8_gpu"


def _edge_secs(calib):
    """32 x 32: stem, an INT8 3x3/2 layer at index 1 (12 -> 20 channels), an INT8 3x3/1 layer of 32 filters behind which a
    2x2/2 max-pool feeds another INT8 layer (32 -> 24: off the tile multiples), float 1x1 layers and a [yolo] head"""
    return [cfgs._net(32, 32, calib),
            cfgs._conv(12, 3),                        # 0 float (index 0)
            cfgs._conv(20, 3, 2),                     # 1 INT8: stride 2 at index 1
            cfgs._conv(32, 3),                        # 2 INT8, pool fused into its epilogue
            ("maxpool", {"size": "2", "stride": "2"}),
            cfgs._conv(24, 3),                        # 4 INT8 (c = 32, n = 24)
            cfgs._conv(40, 3),                        # 5 INT8 (24 -> 40)
            cfgs._conv(16, 1),                        # 6 float (1x1); the [yolo] latch from here on
            cfgs._conv(18, 1, bn=False, act="linear"),
            cfgs._yolo("0,1,2", cfgs.TINY_ANCHORS, 6, classes=1)]


@pytest.fixture(scope="module")
def edge_net(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("edges"))
    # large images and multipliers: every INT8 layer's input has values with |x * m| >= 32768
    cfg, wts = util.write_net(d, "gpu_rule_edges", _edge_secs([2048, 2048, 2 ** 20, 2 ** 20, 2 ** 20, 16, 16]), 43)
    x = cfgs.synthetic_images(3, 3, 32, 32, seed=44) * np.float32(40)
    return cfg, wts, x


@pytest.mark.parametrize("mode", ["fused", "no_tc", "grid2"])
def test_edges_bit_exact(mode, edge_net, monkeypatch):
    import yolo2_light_b200 as yb
    from oracle import port
    cfg, wts, x = edge_net
    if mode == "no_tc":
        monkeypatch.setenv("YB_NO_TC", "1")
    if mode == "grid2":
        monkeypatch.setenv("YB_TC_GRID", "2")
    net = util.load(cfg, wts, 3, quantized=1, precision=yb.YB_PREC_FP32)
    assert _int8_layers(net) == [1, 2, 4, 5]
    net.predict(x, quantized=Q)
    layers = net.layers
    outs = ro.forward(layers, x, Q)
    _assert_bit_exact(net, outs, need=(1, 5))
    # some inputs of the INT8 layers convert differently under the two rules: the saturating conversion ran
    differ = [i for i in _int8_layers(net)
              if not np.array_equal(port.quantize_input(outs[i - 1], layers[i]["input_quant_multipler"]),
                                    ro.quantize_input_gpu(outs[i - 1], layers[i]["input_quant_multipler"]))]
    assert differ == _int8_layers(net), differ
    ops = [(li, k) for li, k, _ in net.profile(quantized=Q)]
    names = {li: nm for li, _, nm in net.op_kernels(quantized=Q)}
    if mode == "no_tc":
        for i in _int8_layers(net):
            assert "SimtInt8Gpu" in (names.get(i) or ""), (i, names.get(i))
    else:
        # layer 2 runs the max-pool and layer 4's conversion in its epilogue
        assert (3, "maxpool") not in ops and (4, "quantize") not in ops, ops
        assert net.tc_plan(2, quantized=Q)["kind"] == "s8_gpu"


def test_rules_coexist_on_one_network(workdir):
    """Predicting with rules 1, 2, 1 on one yb_network leaves rule 1's outputs bit-identical to a fresh network's."""
    cfg, wts = util.model_files("tiny64", workdir)
    x = util.images("tiny64", 2)
    fresh = util.load(cfg, wts, 2, quantized=1)
    fresh.predict(x, quantized=1)
    ref = fresh.detection_outputs()
    net = util.load(cfg, wts, 2, quantized=1)
    net.predict(x, quantized=1)
    net.predict(x, quantized=Q)
    two = net.detection_outputs()
    net.predict(x, quantized=1)
    for i, o in net.detection_outputs().items():
        assert util.bits_equal(o, ref[i]), i
        assert not util.bits_equal(two[i], ref[i]), i


def test_serving_and_multi_gpu(workdir):
    """submit_frames_u8 with rule 2 returns the rows of detect after predict_frames_u8 with rule 2; predict_batch over a
    repeated device list equals the one-GPU call."""
    cfg, wts = util.model_files("tiny64", workdir)
    net = util.load(cfg, wts, 2, quantized=1)
    rng = np.random.default_rng(5)
    frames = [rng.integers(0, 256, (64, 64, 3), dtype=np.uint8), rng.integers(0, 256, (96, 80, 3), dtype=np.uint8)]
    net.predict_frames_u8(frames, quantized=Q)
    exp, ce = net.detect_frames([(f.shape[1], f.shape[0]) for f in frames], 0.05, 0.45, relative=0, max_rows=2048, quantized=Q)
    t = net.submit_frames_u8(frames, 0.05, 0.45, relative=0, max_rows=2048, quantized=Q)
    got, cg, _ = net.collect_detections(t, quantized=Q)
    assert np.array_equal(ce, cg) and int(cg.sum()) > 0
    for b in range(len(frames)):
        assert util.bits_equal(exp[b], got[b]), b

    x = cfgs.synthetic_images(5, 3, 64, 64, seed=8)
    one = util.load(cfg, wts, 2, quantized=1)
    r1 = one.predict_batch(x, 1, quantized=Q)
    rep = util.load(cfg, wts, 2, quantized=1)
    rep.set_devices([0, 0])
    r2 = rep.predict_batch(x, 2, quantized=Q)
    assert r1.keys() == r2.keys()
    for i in r1:
        assert util.bits_equal(r1[i], r2[i]), i


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref not built")
def test_true_dropin_gpu_rule_behind_reference_host_code(workdir):
    """The reference's own host code parses, loads, folds and quantises; the glue runs the network with the GPU rule on the
    reference layers' own l.quantized (passed through yb_layer_desc.quantized).  The reference harness reaches the glue's rule
    argument through network_predict_b200_batch(net, ..., quantized), which forwards the value its network was parsed with, so
    the cfg is parsed with quantized = 2 -- the reference treats every non-zero value alike, and its l.quantized flags are
    those of a quantized = 1 parse.  The last layer's yolo tensor is the oracle's GPU rule within the tf32 bar: the glue runs
    the default precision, where the float layers behind the INT8 ones take tf32."""
    from oracle import port, ref
    cfg, wts = util.model_files("tiny64", workdir)
    x = util.images("tiny64", 1)
    rnet = ref.RefNet(cfg, wts, 1, Q, 7, kind="dropin")
    assert rnet.layers[-1]["type_name"] == "YOLO"
    mine = util.load(cfg, wts, 1, quantized=1)
    assert [i for i, L in enumerate(rnet.layers) if L["type_name"] == "CONVOLUTIONAL" and L["quantized"]] == _int8_layers(mine)
    got = rnet.predict_b200_batch(x, 1)
    outs = ro.forward(mine.layers, x, Q)
    err = util.rel_l2(got, outs[-1].reshape(got.shape))
    assert err <= 1e-3, err
    # the CPU rule on the same layers is farther away than that: the GPU rule ran
    cpu = port.run_network(mine.layers, x, quantized=True)
    assert util.rel_l2(got, cpu[-1].reshape(got.shape)) > err


def test_yolov3_608_batch2(tmp_path_factory):
    """yolov3 608, batch 2, with the layer-1 quirk (the 3x3/2 layer at index 1 is INT8): bit-identical to the oracle at
    YB_PREC_FP32, within rel-L2 1e-3 of that at the default precision."""
    import yolo2_light_b200 as yb
    d = str(tmp_path_factory.mktemp("v3_608"))
    cfg, wts = util.write_net(d, "v3_608", cfgs.yolov3(608, 608), 45)
    x = cfgs.synthetic_images(2, 3, 608, 608, seed=46)
    exact = util.load(cfg, wts, 2, quantized=1, precision=yb.YB_PREC_FP32)
    q = _int8_layers(exact)
    assert len(q) == 26 and q[0] == 1 and max(q) == 78
    exact.predict(x, quantized=Q)
    ref_out = exact.detection_outputs()
    outs = ro.forward(exact.layers, x, Q)
    for i, o in ref_out.items():
        assert util.bits_equal(o, outs[i].reshape(o.shape)), i
    fast = util.load(cfg, wts, 2, quantized=1)
    fast.predict(x, quantized=Q)
    for i, o in fast.detection_outputs().items():
        err = util.rel_l2(o, ref_out[i])
        assert err <= 1e-3, (i, err)
    # the 48 float convolutions but the stem run on tf32, and nothing else does
    convs = [i for i, l in enumerate(fast.layers) if l["type_name"] == "CONVOLUTIONAL"]
    tf32 = [i for i in convs if fast.tc_plan(i, quantized=Q).get("kind") == "tf32"]
    assert tf32 == [i for i in convs if i > 0 and i not in q] and len(tf32) == 48, tf32
