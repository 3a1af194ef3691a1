"""256-filter tiles of the register-accumulator convolution kernel.  The automatic filter-tile width picks 256 only where
it saves waves, which the small test grids never do, so YB_TC_BN=256 forces it here: full and masked (320 = 256 + 64)
tiles, and a fused shortcut on a 256-wide tile."""
import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import bf16_round, tcnet, widenet
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu


def test_tc_bn256_every_layer_vs_oracle(workdir, monkeypatch):
    import yolo2_light_b200 as yb
    from oracle import port
    monkeypatch.setenv("YB_TC_BN", "256")
    net = util.load(*util.write_net(workdir, "tcnet64bn256", tcnet(64), 21), 2, precision=yb.YB_PREC_BF16_TC, fuse=0)
    x = cfgs.synthetic_images(2, 3, 64, 64, seed=5)
    net.predict(x)
    kinds = util.profile_kinds(net)
    layers = net.layers
    got = [net.fetch_layer(i) for i in range(net.n)]
    for i, l in enumerate(layers):
        if l["type_name"] != "CONVOLUTIONAL" or i == 0:
            continue
        assert "conv_tc" in kinds.get(i, []), i
        w = bf16_round(l["weights"])
        exp = port.conv_fp32(got[i - 1], w, l["biases"], l["n"], l["size"], l["stride"], l["pad"], l["activation"])
        if l["activation"] != 3:
            exp = bf16_round(exp)
        assert util.rel_l2(got[i], exp) <= 5e-4, i


@pytest.mark.parametrize("bn", ["256", None])
def test_tc_wide_fused_shortcut_vs_f32_oracle(bn, workdir, monkeypatch):
    from oracle import port
    if bn:
        monkeypatch.setenv("YB_TC_BN", bn)
    cfg, wts = util.write_net(workdir, "widenet", widenet(), 31)
    x = cfgs.synthetic_images(2, 3, 32, 32, seed=8)
    outs = []
    for fuse in (0, 1):
        net = util.load(cfg, wts, 2, fuse=fuse)
        net.predict(x)
        outs.append({i: o.copy() for i, o in net.detection_outputs().items()})
        if fuse:
            exp = [port.run_network(net.layers, x[b:b + 1]) for b in range(2)]
    for i, o in outs[1].items():
        e = np.concatenate([exp[b][i] for b in range(2)], 0).reshape(o.shape)
        assert util.rel_l2(o, e) <= 3e-3, (i, util.rel_l2(o, e))
        assert util.rel_l2(o, outs[0][i]) <= 2e-3, i   # residual add before vs after bf16 rounding
