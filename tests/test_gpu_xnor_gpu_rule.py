"""The GPU build's XNOR arithmetic (YB_XNOR_GPU) on the H100: path A (the bit GEMM's FMA epilogue and folded shortcut, every
geometry at c % 32 == 0) and path B (zero-padded +-1 layers below 32 channels), checked bit for bit against the restatement
in tests/rule_oracle.py, per layer and on the final tensors.  GPU box only."""
import numpy as np
import pytest

import rule_oracle as ro
import ybtest_util as util
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu


def _edge_secs():
    """32 x 32: a stem and max-pool in front of a 16-channel XNOR layer (path B on the s8 wgmma), a relu float layer whose
    exact zeros (+0 and -0) feed a second path-B layer, path-A layers at c = 32 (max-pool fused behind it), 64 and 128, a
    linear path-A layer with a same-shape leaky [shortcut] behind it, path A at stride 2, at 1x1 and with a logistic
    activation, and a [yolo] head.  Parsed with quantized = 1 the 3x3/1 non-linear layers 2-8 are the GPU INT8 rule's
    l.quantized layers; the [yolo] latch leaves layer 13 to XNOR."""
    x = lambda n, size=3, stride=1, act="leaky": cfgs._conv(n, size, stride, act=act, xnor=1)
    return [cfgs._net(32, 32),
            cfgs._conv(16, 3),                                     # 0 stem
            ("maxpool", {"size": "2", "stride": "2"}),             # 1
            x(32),                                                 # 2 B (c = 16)
            cfgs._conv(16, 3, act="relu"),                         # 3 float, exact zeros
            x(32),                                                 # 4 B (c = 16), zero inputs
            x(32),                                                 # 5 A (c = 32)
            ("maxpool", {"size": "2", "stride": "2"}),             # 6
            x(64),                                                 # 7 A (c = 32)
            x(128),                                                # 8 A (c = 64)
            x(128, act="linear"),                                  # 9 A (c = 128), shortcut folded
            ("shortcut", {"from": "-2", "activation": "leaky"}),   # 10 from 8, activation not applied
            x(128, 3, 2),                                          # 11 A, stride 2
            x(64, 1),                                              # 12 A, 1x1
            x(32, act="logistic"),                                 # 13 A, logistic
            cfgs._conv(18, 1, bn=False, act="linear"),             # 14
            cfgs._yolo("0,1,2", cfgs.TINY_ANCHORS, 6, classes=1)]  # 15


@pytest.fixture(scope="module")
def edge_net(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("xnor_gpu_edges"))
    cfg, wts = util.write_net(d, "xnor_gpu_edges", _edge_secs(), 61)
    x = cfgs.synthetic_images(2, 3, 32, 32, seed=62)
    return cfg, wts, x


def _load(cfg, wts, batch, quantized=0, **kw):
    import yolo2_light_b200 as yb
    net = util.load(cfg, wts, batch, quantized=quantized, **kw)
    net.set_xnor_rule(yb.YB_XNOR_GPU)
    return net


def _check(net, outs, q, upto=None):
    """every materialised layer (below `upto`) and every detection tensor bit for bit; returns the fetched layers"""
    got = util.fetch_all(net, q)
    for i, o in got.items():
        if upto is None or i < upto:
            assert util.bits_equal(o, np.asarray(outs[i]).reshape(o.shape)), i
    if upto is None:
        for i, o in net.detection_outputs().items():
            assert util.bits_equal(o, np.asarray(outs[i]).reshape(o.shape)), i
    return got


@pytest.mark.parametrize("mode", ["fused", "xnor_tc0", "grid1", "no_pool_fuse", "unfused"])
def test_edges_bit_exact(mode, edge_net, monkeypatch):
    """quantized = 0, YB_PREC_FP32: every layer and the yolo tensor are the restatement's, on every kernel path the
    switches select; the folded shortcut and the fused max-pools are where the plan puts them."""
    import yolo2_light_b200 as yb
    cfg, wts, x = edge_net
    env = {"xnor_tc0": ("YB_XNOR_TC", "0"), "grid1": ("YB_TC_GRID", "1"), "no_pool_fuse": ("YB_NO_POOL_FUSE", "1")}
    if mode in env:
        monkeypatch.setenv(*env[mode])
    net = _load(cfg, wts, 2, precision=yb.YB_PREC_FP32, fuse=0 if mode == "unfused" else None)
    assert net.get_info("xnor_rule") == yb.YB_XNOR_GPU
    net.predict(x)
    layers = net.layers
    A, B = "xnor_gpu", "pm1z_gpu"
    assert util.xnor_gpu_layers(layers) == {2: B, 4: B, 5: A, 7: A, 8: A, 9: A, 11: A, 12: A, 13: A}
    outs = ro.forward(layers, x, 0, ro.XNOR_GPU)
    got = _check(net, outs, 0)
    assert {2, 4, 9, 10, 11, 12, 13} <= set(got)
    # the GPU build's arithmetic, not the CPU build's
    from oracle import port
    cpu = port.run_network(layers, x[:1])
    assert not util.bits_equal(cpu[4], outs[4][:1]) and not util.bits_equal(cpu[10], outs[10][:1])
    if mode == "fused":
        assert net.tc_plan(2)["kind"] == "pm1z_gpu" and net.tc_plan(9)["kind"] == "xnor_gpu"
        assert net.tc_plan(5)["kind"] == "xnor_gpu" and 6 not in got   # max-pool in layer 5's epilogue
    if mode == "xnor_tc0":
        for i in (2, 4, 5, 7, 8, 9, 13):
            assert net.tc_plan(i) == {}, i


def test_edges_default_precision_and_counts(edge_net):
    """Default precision: every layer in front of the head is bit-exact (the XNOR networks keep f32 activations), the yolo
    tensor within rel-L2 1e-3 of the restatement (the head runs on tf32); the raw results are the restatement's dot / s."""
    cfg, wts, x = edge_net
    net = _load(cfg, wts, 2, fuse=0, keep_counts=True)
    net.predict(x)
    layers = net.layers
    outs = ro.forward(layers, x, 0, ro.XNOR_GPU)
    _check(net, outs, 0, upto=14)
    for i, o in net.detection_outputs().items():
        assert util.rel_l2(o, outs[i].reshape(o.shape)) <= 1e-3, i
    for i, arith in util.xnor_gpu_layers(layers).items():
        fn = ro.bin_dot if arith == "xnor_gpu" else ro.pm1z_sum
        L = layers[i]
        raw = fn(outs[i - 1], L["weights"], L["n"], L["size"], L["stride"], L["pad"])
        cnt = net.fetch_counts(i)
        assert np.array_equal(cnt, (raw + L["size"] ** 2 * L["c"]) // 2 if arith == "xnor_gpu" else raw), i


@pytest.mark.parametrize("precision", ["fp32", "default"])
def test_gpu_int8_rule_with_xnor_layers(precision, edge_net):
    """quantized = 2 completes network_predict_gpu_cudnn_quantized: layers 2-8 run INT8 (l.quantized), the others by the
    XNOR rule; bit-exact at YB_PREC_FP32, the layers in front of the tf32 head bit-exact at the default precision."""
    import yolo2_light_b200 as yb
    cfg, wts, x = edge_net
    net = _load(cfg, wts, 2, quantized=1, precision=yb.YB_PREC_FP32 if precision == "fp32" else None, fuse=0)
    layers = net.layers
    assert [i for i, L in enumerate(layers) if L["type_name"] == "CONVOLUTIONAL" and L["quantized"]] == [2, 3, 4, 5, 7, 8]
    assert util.xnor_gpu_layers(layers, quantized=2) == {9: "xnor_gpu", 11: "xnor_gpu", 12: "xnor_gpu", 13: "xnor_gpu"}
    net.predict(x, quantized=2)
    outs = ro.forward(layers, x, 2, ro.XNOR_GPU)
    _check(net, outs, 2, upto=None if precision == "fp32" else 14)
    with pytest.raises(yb.YbError, match="quantized = 1"):
        net.predict(x, quantized=1)


def test_xnor64_both_precisions(workdir):
    """xnor64 (tiny-yolo-obj_xnor slimmed, 64 x 64, batch 3): every layer in front of the [region] bit-exact at YB_PREC_FP32,
    the region tensor within a few ulps (its logistic and softmax use the device's exponential); at the default precision
    the region tensor is within the tf32 bar of that."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("xnor64", workdir)
    x = util.images("xnor64", 3)
    exact = _load(cfg, wts, 3, precision=yb.YB_PREC_FP32)
    exact.predict(x)
    outs = ro.forward(exact.layers, x, 0, ro.XNOR_GPU)
    _check(exact, outs, 0, upto=15)
    region = exact.detection_outputs()[15]
    assert np.allclose(region, outs[15].reshape(region.shape), rtol=2.0 ** -20, atol=0)
    fast = _load(cfg, wts, 3)
    fast.predict(x)
    ref = exact.detection_outputs()
    for i, o in fast.detection_outputs().items():
        assert util.rel_l2(o, ref[i]) <= 1e-3, i


def test_serving_and_batch_match_predict(edge_net):
    """submit / collect and yb_network_predict_batch (a partial last batch, and two replicas on one device) give
    yb_network_predict's tensors bit for bit."""
    cfg, wts, x = edge_net
    net = _load(cfg, wts, 2)
    net.predict(x)
    ref = {i: o.copy() for i, o in net.detection_outputs().items()}
    t = net.submit(x)
    got = net.collect(t)
    for i, o in got.items():
        assert util.bits_equal(o, ref[i]), i
    x3 = np.concatenate([x, x[:1]], 0)
    one = _load(cfg, wts, 2)
    r1 = one.predict_batch(x3, 1)
    rep = _load(cfg, wts, 2)
    rep.set_devices([0, 0])
    r2 = rep.predict_batch(x3, 2)
    for i in r1:
        assert util.bits_equal(r1[i][:2].reshape(ref[i].shape), ref[i]), i
        assert util.bits_equal(r1[i], r2[i]), i
        assert util.bits_equal(r1[i][2], r1[i][0]), i


def test_rules_coexist_on_one_network(workdir):
    """CPU, GPU, CPU XNOR rule on one yb_network (xnor64): the CPU rule's tensors are a fresh network's, the GPU rule's
    differ."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("xnor64", workdir)
    x = util.images("xnor64", 2)
    fresh = util.load(cfg, wts, 2)
    fresh.predict(x)
    ref = {i: o.copy() for i, o in fresh.detection_outputs().items()}
    assert fresh.get_info("xnor_rule") == yb.YB_XNOR_CPU
    net = util.load(cfg, wts, 2)
    net.predict(x)
    net.set_xnor_rule(yb.YB_XNOR_GPU)
    net.predict(x)
    gpu = {i: o.copy() for i, o in net.detection_outputs().items()}   # host views of the engine's outputs
    net.set_xnor_rule(yb.YB_XNOR_CPU)
    net.predict(x)
    for i, o in net.detection_outputs().items():
        assert util.bits_equal(o, ref[i]), i
        assert not util.bits_equal(gpu[i], ref[i]), i


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref not built")
def test_true_dropin_behind_reference_host_code(workdir, monkeypatch):
    """The reference's own host code parses, loads and prepares xnor64, and the drop-in glue runs it in network_predict_b200's
    slot, with the GPU XNOR rule chosen through YB_XNOR_RULE=1: the glue's networks start with it, whichever glue build the
    host links.  The region tensor is the restatement's within the tf32 bar of the head, and farther from the CPU build's
    XNOR arithmetic than that."""
    from oracle import port, ref
    cfg, wts = util.model_files("xnor64", workdir)
    x = util.images("xnor64", 1)
    monkeypatch.setenv("YB_XNOR_RULE", "1")
    rnet = ref.RefNet(cfg, wts, 1, 0, 7, kind="dropin")
    got = rnet.predict_b200_batch(x, 1)
    monkeypatch.delenv("YB_XNOR_RULE")
    mine = util.load(cfg, wts, 1)
    outs = ro.forward(mine.layers, x, 0, ro.XNOR_GPU)
    err = util.rel_l2(got, outs[-1].reshape(got.shape))
    assert err <= 1e-3, err
    cpu = port.run_network(mine.layers, x)
    assert util.rel_l2(got, cpu[-1].reshape(got.shape)) > err


def test_initial_rule_from_the_environment(workdir, monkeypatch):
    """YB_XNOR_RULE=1 starts a network (parsed or built from layer descriptions) on the GPU XNOR rule, bit-identical to one
    switched by yb_network_set_xnor_rule; yb_network_set_xnor_rule overrides it."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("xnor64", workdir)
    x = util.images("xnor64", 2)
    switched = _load(cfg, wts, 2)
    switched.predict(x)
    ref = {i: o.copy() for i, o in switched.detection_outputs().items()}
    monkeypatch.setenv("YB_XNOR_RULE", "1")
    net = util.load(cfg, wts, 2)
    assert net.get_info("xnor_rule") == yb.YB_XNOR_GPU
    net.predict(x)
    for i, o in net.detection_outputs().items():
        assert util.bits_equal(o, ref[i]), i
    net.set_xnor_rule(yb.YB_XNOR_CPU)
    assert net.get_info("xnor_rule") == yb.YB_XNOR_CPU
