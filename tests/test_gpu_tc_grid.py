"""Persistent schedule of the tensor-core convolutions with many work items per CTA.  On the small test grids every CTA
gets about one work item, so YB_TC_GRID caps the grid at 1, 2 and 3 CTAs: each CTA then walks many work items (odd counts
included), reuses its epilogue staging buffers from tile to tile and flips every barrier phase many times.  Every filter-tile
width of k_conv_tc_reg, with and without fused shortcuts, must give bit-identical layer outputs to the full grid."""
import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import tcnet, widenet
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu

NETS = {"widenet": (widenet, 32, 31, 8), "tcnet": (lambda: tcnet(64), 64, 21, 5)}


@pytest.mark.parametrize("bn", ["32", "64", "128", "256"])
@pytest.mark.parametrize("name", list(NETS))
def test_tc_small_grid_bit_equal_to_full_grid(name, bn, workdir, monkeypatch):
    from oracle import port
    build, size, wseed, xseed = NETS[name]
    cfg, wts = util.write_net(workdir, f"{name}_grid", build(), wseed)
    x = cfgs.synthetic_images(2, 3, size, size, seed=xseed)
    monkeypatch.setenv("YB_TC_BN", bn)
    exp = None
    for fuse in (0, 1):
        ref = None
        for grid in (None, "1", "2", "3"):
            if grid:
                monkeypatch.setenv("YB_TC_GRID", grid)
            else:
                monkeypatch.delenv("YB_TC_GRID", raising=False)
            net = util.load(cfg, wts, 2, fuse=fuse)
            net.predict(x)
            got = util.fetch_all(net)
            # with fusion on, a conv fused into its shortcut has no output of its own
            assert fuse or len(got) == net.n, (fuse, sorted(got))
            dets = {i: o.copy() for i, o in net.detection_outputs().items()}
            if exp is None:
                exp = [port.run_network(net.layers, x[b:b + 1]) for b in range(2)]
            for i, o in dets.items():
                e = np.concatenate([exp[b][i] for b in range(2)], 0).reshape(o.shape)
                assert util.rel_l2(o, e) <= 3e-3, (fuse, grid, i, util.rel_l2(o, e))
            if ref is None:
                ref = got
                continue
            assert got.keys() == ref.keys()
            for i in got:
                assert np.array_equal(got[i], ref[i]), (fuse, grid, i)
