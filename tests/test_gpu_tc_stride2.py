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
from test_gpu_tc import _files, bf16_round
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu

SHAPES = [((152, 152), 3), ((232, 136), 3)]
TW = {(152, 152): (16, 1, 2), (232, 136): (4, 2, 4)}   # the tile width of stride-2 layers 1, 3 and 5


def s2chain():
    c = cfgs._conv
    return [cfgs._net(64, 64),
            c(32, 3),                   # 0 stem
            c(64, 3, 2),                # 1 s2, C=32
            c(64, 3),                   # 2 s1 over layer 1's borders
            c(128, 3, 2),               # 3 s2
            c(128, 3),                  # 4
            c(256, 3, 2),               # 5 s2, up to 256 filters per tile
            c(256, 3),                  # 6
            c(255, 1, bn=False, act="linear"),
            cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9)]


def _net(workdir, hw, batch, seed):
    import yolo2_light_b200 as yb
    h, w = hw
    secs = s2chain()
    secs[0][1]["height"], secs[0][1]["width"] = str(h), str(w)
    cfg, wts = _files(workdir, f"s2chain{h}x{w}", secs, seed)
    net = yb.load_network(cfg, wts, batch=batch)
    net.set_precision(yb.YB_PREC_BF16_TC)
    net.set_option("fuse", 0)
    return net, cfgs.synthetic_images(batch, 3, h, w, seed=seed + 1)


@pytest.mark.parametrize("bn", ["32", "64", "128", "256"])
@pytest.mark.parametrize("hw,batch", SHAPES)
def test_tc_stride2_reg_every_layer_vs_oracle(hw, batch, bn, workdir, monkeypatch):
    from oracle import port
    monkeypatch.setenv("YB_TC_BN", bn)
    net, x = _net(workdir, hw, batch, 41)
    net.predict(x)
    kinds = {}
    for li, kind, _ in net.profile():
        kinds.setdefault(li, []).append(kind)
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
