"""Stride-2 convolutions in k_conv_tc_reg.  Their tiles walk the input's merged half rows (OH + 1 per image), so on small
grids most half tiles straddle two images and are stored one tile row at a time.  Each stride-2 layer is followed by a 3x3
stride-1 layer, which reads the stride-2 output's zero border: a border row stored with data shows up in its result.

Shapes (batch, output sizes, tile width TW picked by the plan):
  152x152, batch 3: 76x76 (TW 16), 38x38 (TW 1), 19x19 (TW 2)
  232x136, batch 3: 116x68 (TW 4), 58x34 (TW 2), 29x17 (TW 4)
Every filter-tile width is forced with YB_TC_BN (capped by the filters)."""
import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import bf16_round, s2chain
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu

SHAPES = [((152, 152), 3), ((232, 136), 3)]
TW = {(152, 152): (16, 1, 2), (232, 136): (4, 2, 4)}   # the tile width of stride-2 layers 1, 3 and 5


def _net(workdir, hw, batch, seed):
    import yolo2_light_b200 as yb
    h, w = hw
    secs = s2chain()
    secs[0][1]["height"], secs[0][1]["width"] = str(h), str(w)
    net = util.load(*util.write_net(workdir, f"s2chain{h}x{w}_{seed}", secs, seed), batch, precision=yb.YB_PREC_BF16_TC, fuse=0)
    return net, cfgs.synthetic_images(batch, 3, h, w, seed=seed + 1)


@pytest.mark.parametrize("bn", ["32", "64", "128", "256"])
@pytest.mark.parametrize("hw,batch", SHAPES)
def test_tc_stride2_reg_every_layer_vs_oracle(hw, batch, bn, workdir, monkeypatch):
    from oracle import port
    monkeypatch.setenv("YB_TC_BN", bn)
    net, x = _net(workdir, hw, batch, 41)
    net.predict(x)
    kinds = util.profile_kinds(net)
    layers = net.layers
    got = [net.fetch_layer(i) for i in range(net.n)]
    for i, tw in zip((1, 3, 5), TW[hw]):
        p = net.tc_plan(i)
        # BN 32 with TW 1 takes TW 2: a one-row store of a straddling half tile must start 128-byte aligned
        assert p["kernel"] == "k_conv_tc_reg" and p["TW"] == (2 if tw == 1 and p["BN"] == 32 else tw), (hw, bn, i, p)
    for i in range(1, 7):
        assert "conv_tc" in kinds.get(i, []), (i, kinds.get(i))
        l = layers[i]
        exp = bf16_round(port.conv_fp32(got[i - 1], bf16_round(l["weights"]), l["biases"], l["n"], l["size"], l["stride"], l["pad"],
                                        l["activation"]))
        err = util.rel_l2(got[i], exp)
        assert err <= 5e-4, (hw, bn, i, err)


@pytest.mark.parametrize("bn", ["32", "64", "128", "256"])
def test_tc_stride2_reg_small_grid_bit_equal(bn, workdir, monkeypatch):
    """1, 2 and 3 CTAs walk many work items each, straddling and one-image half tiles mixed: bit-equal to the full grid."""
    monkeypatch.setenv("YB_TC_BN", bn)
    hw, batch = SHAPES[0]
    ref = None
    for grid in (None, "1", "2", "3"):
        if grid:
            monkeypatch.setenv("YB_TC_GRID", grid)
        else:
            monkeypatch.delenv("YB_TC_GRID", raising=False)
        net, x = _net(workdir, hw, batch, 43)
        net.predict(x)
        got = [net.fetch_layer(i) for i in range(7)]
        if ref is None:
            ref = got
            continue
        for i in range(7):
            assert np.array_equal(got[i], ref[i]), (bn, grid, i)
