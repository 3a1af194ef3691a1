"""The GPU build's XNOR arithmetic (YB_XNOR_GPU, yb_network_set_xnor_rule) on the host side: the per-layer path choice and
the rejections on the reference's parsed layers, the restatement's epilogue at its edges, its dot against the CPU oracle's
popcounts, and the loud failure of every new entry point without a device."""
import os

import numpy as np
import pytest

import rule_oracle as ro
import ybtest_util as util
from yolo2_light_b200 import cfgs

F32 = np.float32
XNOR_CFG = os.path.join(util.GOLDEN, "assets", "tiny-yolo-obj_xnor.cfg")


def _xconv(filters, size=3, stride=1, act="leaky"):
    return cfgs._conv(filters, size, stride, act=act, xnor=1)


def _secs(*body, w=16, h=16):
    return [cfgs._net(w, h)] + list(body)


def _parsed(secs, tmp_path, name):
    """the reference's parsed layers of `secs` where the reference is built, else ours"""
    cfg = cfgs.write_cfg(secs, str(tmp_path / (name + ".cfg")))
    if util.have_ref():
        from oracle import ref
        return ref.RefNet(cfg, None, 1, 0, 0).layers
    import yolo2_light_b200 as yb
    return yb.parse_network_cfg(cfg, 1, 0).layers


def test_paths_of_tiny_yolo_obj_xnor():
    """tiny-yolo-obj_xnor: the 16-channel XNOR layer behind the stem's max-pool is path B (pm1z_gpu), the wider ones path A
    (xnor_gpu)."""
    if util.have_ref():
        from oracle import ref
        layers = ref.RefNet(XNOR_CFG, None, 1, 0, 0).layers
    else:
        import yolo2_light_b200 as yb
        layers = yb.parse_network_cfg(XNOR_CFG, 1, 0).layers
    paths = util.xnor_gpu_layers(layers)
    xnor = [i for i, L in enumerate(layers) if L["type_name"] == "CONVOLUTIONAL" and L["xnor"]]
    assert sorted(paths) == xnor
    assert {i: p for i, p in paths.items() if p == "pm1z_gpu"} == {i: "pm1z_gpu" for i in xnor if layers[i]["c"] < 32}
    assert [paths[i] for i in xnor].count("pm1z_gpu") == 1 and layers[xnor[0]]["c"] == 16


@pytest.mark.parametrize("case", ["c48", "sc_pathB", "sc_logistic", "sc_ok", "s2_1x1"])
def test_paths_and_rejections_of_small_cfgs(case, tmp_path):
    sc = ("shortcut", {"from": "-2", "activation": "leaky"})
    if case == "c48":                     # c >= 32, c % 32 != 0: no convolution in the reference
        secs, want = _secs(cfgs._conv(48, 3), _xconv(32)), "c = 48"
    elif case == "sc_pathB":              # the shortcut the GPU build blanks, never written by path B
        secs, want = _secs(cfgs._conv(16, 3), _xconv(16), sc), "never written"
    elif case == "sc_logistic":
        secs, want = _secs(cfgs._conv(32, 3), _xconv(32, act="logistic"), sc), "non-leaky"
    elif case == "sc_ok":
        secs, want = _secs(cfgs._conv(32, 3), _xconv(32), sc), {1: "xnor_gpu"}
    else:
        secs, want = _secs(cfgs._conv(32, 3), _xconv(64, 3, 2), _xconv(64, 1), _xconv(8, 3)), {1: "xnor_gpu", 2: "xnor_gpu", 3: "xnor_gpu"}
    layers = _parsed(secs, tmp_path, case)
    if isinstance(want, dict):
        assert util.xnor_gpu_layers(layers) == want
    else:
        with pytest.raises(ro.Rejected, match=want):
            util.xnor_gpu_layers(layers)


def test_int8_layers_of_the_gpu_int8_rule_keep_no_xnor_path():
    layers = [dict(type_name="CONVOLUTIONAL", xnor=1, quantized=1, c=32, activation=7),
              dict(type_name="CONVOLUTIONAL", xnor=1, quantized=0, c=32, activation=7)]
    assert util.xnor_gpu_layers(layers, quantized=2) == {1: "xnor_gpu"}
    assert util.xnor_gpu_layers(layers) == {0: "xnor_gpu", 1: "xnor_gpu"}


def test_fmaf_is_correctly_rounded():
    """The vectorised fmaf against exact rationals, on random values and on products that sit on a float32 midpoint of
    the sum, where fmaf and the two-rounding expression differ."""
    rng = np.random.default_rng(3)
    a = rng.integers(-4000, 4000, 3000).astype(F32)
    b = rng.uniform(0.001, 2, 3000).astype(F32)
    c = rng.normal(0, 50, 3000).astype(F32)
    got = ro.fmaf_f32(a, b, c)
    exp = np.array([ro.fmaf_exact(*t) for t in zip(a, b, c)], F32)
    assert util.bits_equal(got, exp)
    two = ((a * b).astype(F32) + c).astype(F32)
    assert not util.bits_equal(got, two)
    # dot * mean lands between two float32 values next to 1.0: the separately rounded product loses what fmaf keeps
    m = F32(1.0) + F32(2.0 ** -23)
    a2, b2, c2 = F32(3.0), m, F32(-3.0)
    assert ro.fmaf_f32(a2, b2, c2) == ro.fmaf_exact(a2, b2, c2) == F32(3 * 2.0 ** -23)
    assert F32(F32(a2 * b2) + c2) != F32(3 * 2.0 ** -23)
    # a tie of the double sum decided by the TwoSum error
    a3, b3, c3 = F32(1.0), F32(1.0 + 2.0 ** -23), F32(2.0 ** -24 + 2.0 ** -48)
    assert ro.fmaf_f32(a3, b3, c3) == ro.fmaf_exact(a3, b3, c3)


def test_epilogue_edges():
    """Leaky in float (0.1f * y, not the double 0.1 * y), -0 through leaky, and the path-B sign: x >= 0, so +0 and -0 are +1
    while path A's bit is x > 0."""
    from oracle import port
    y = np.array([-0.0, 0.0, -1e-30, -3.3333333, 7.0], F32)
    got = ro.act_gpu(y, port.LEAKY)
    assert got[0] == 0 and np.signbit(got[0]) and not np.signbit(got[1])
    assert got[3] == F32(0.1) * F32(-3.3333333)
    v = np.arange(1, 20000, dtype=F32) * F32(-0.37)
    assert not util.bits_equal(ro.act_gpu(v, port.LEAKY), (0.1 * v.astype(np.float64)).astype(F32))
    x = np.array([[[[0.0, -0.0, 1.0, -1.0]]]], F32)
    w = np.ones(1, F32)
    assert ro.pm1z_sum(x, w, 1, 1, 1, 0).ravel().tolist() == [1, 1, 1, -1]
    assert ro.bin_dot(x, w, 1, 1, 1, 0).ravel().tolist() == [-1, -1, 1, -1]
    # out-of-image taps: -1 on path A, 0 on path B
    ones = np.ones((1, 1, 2, 2), F32)
    assert ro.bin_dot(ones, np.ones(9, F32), 1, 3, 1, 1).ravel().tolist() == [-1] * 4
    assert ro.pm1z_sum(ones, np.ones(9, F32), 1, 3, 1, 1).ravel().tolist() == [4] * 4


@pytest.mark.parametrize("c", [32, 64])
def test_path_a_dot_is_the_cpu_oracles(c):
    """dot = 2*count - K equals the CPU oracle's XNOR popcounts at 3x3/1/1, and its output differs from the CPU epilogue
    only by the FMA."""
    from oracle import port
    rng = np.random.default_rng(c)
    n = 24
    x = rng.normal(0, 1, (2, c, 7, 9)).astype(F32)
    x[0, 0, 0, :3] = 0.0
    L = dict(n=n, size=3, stride=1, pad=1, activation=port.LINEAR, weights=rng.normal(0, 1, n * c * 9).astype(F32),
             biases=rng.normal(0, 1, n).astype(F32), mean_arr=rng.uniform(0.01, 1, n).astype(F32))
    y, dot = ro.conv_xnor_a(x, L, want_raw=True)
    cpu, counts = port.conv_xnor(x, L["weights"], L["biases"], L["mean_arr"], n, 3, port.LINEAR, want_counts=True)
    assert np.array_equal(dot, 2 * counts - c * 9)
    # one rounding of the product apart: within an ulp of its magnitude
    mag = np.abs(dot * L["mean_arr"].reshape(1, n, 1, 1).astype(np.float64)) + np.abs(L["biases"]).reshape(1, n, 1, 1)
    assert (np.abs(y.astype(np.float64) - cpu) <= mag * 2.0 ** -23).all()
    assert not util.bits_equal(y, cpu)


def test_new_entry_points_fail_loudly_without_a_device(workdir):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("xnor64", workdir)
    net = yb.load_network(cfg, wts, batch=1, quantized=1)
    x = util.images("xnor64", 1)
    net.set_xnor_rule(yb.YB_XNOR_GPU)
    with pytest.raises(yb.YbError, match="bad XNOR rule"):
        net.set_xnor_rule(2)
    calls = [lambda: net.predict(x),
             lambda: net.predict(x, quantized=2),
             lambda: yb.network_predict_b200(net, x),
             lambda: yb.network_predict_b200_cudnn_quantized(net, x),
             lambda: net.submit(x),
             lambda: net.predict_batch(x, 1),
             lambda: net.fetch_layer(2),
             lambda: net.tc_plan(4)]
    for f in calls:
        with pytest.raises(yb.YbError, match="no CUDA device|0 visible"):
            f()
    assert net.get_info("xnor_rule") == -1                       # the engine facts report failure as -1
    assert "no CUDA device" in yb.lib().yb_last_error().decode()


def test_initial_rule_from_the_environment_is_checked(workdir, monkeypatch):
    """YB_XNOR_RULE names a network's initial rule: "0" and "1" create networks, any other value fails the creation."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("xnor64", workdir)
    for v in ("0", "1"):
        monkeypatch.setenv("YB_XNOR_RULE", v)
        assert yb.load_network(cfg, wts, batch=1).n > 0
    for v in ("2", "gpu", ""):
        monkeypatch.setenv("YB_XNOR_RULE", v)
        with pytest.raises(yb.YbError, match="YB_XNOR_RULE"):
            yb.parse_network_cfg(cfg, 1, 0)
