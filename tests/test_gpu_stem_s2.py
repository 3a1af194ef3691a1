"""The tensor-core stem fused with the 3x3 / stride-2 convolution that reads it (k_stem_s2_tc): the stem output stays in
shared memory.  Fused and unfused runs (YB_NO_STEM_S2_FUSE=1) must agree bit for bit on every materialised layer and every
detection tensor, from f32 images and from 8-bit frames, on layer-1 outputs that are not a multiple of the 16 x 8 tile and on
the full 608^2 yolov3; layer 1 is checked against the f32 oracle, and small persistent grids against the full grid."""
import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import bf16_round, s2chain, widenet
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu

NETS = {"s2chain": s2chain, "widenet": widenet}
CASES = [("s2chain", (64, 64), 2), ("s2chain", (96, 160), 3), ("s2chain", (80, 48), 5), ("s2chain", (232, 136), 3),
         ("s2chain", (608, 32), 1), ("widenet", (64, 64), 2), ("widenet", (96, 160), 3), ("widenet", (80, 48), 5),
         ("widenet", (232, 136), 3), ("widenet", (608, 32), 1)]


def _files_for(workdir, name, hw):
    h, w = hw
    secs = NETS[name]()
    secs[0][1]["height"], secs[0][1]["width"] = str(h), str(w)
    return util.write_net(workdir, f"stems2_{name}{h}x{w}", secs, 51)


def _run(cfg, wts, batch, x, monkeypatch, fused, u8=False):
    import yolo2_light_b200 as yb
    if fused:
        monkeypatch.delenv("YB_NO_STEM_S2_FUSE", raising=False)
    else:
        monkeypatch.setenv("YB_NO_STEM_S2_FUSE", "1")
    net = util.load(cfg, wts, batch, precision=yb.YB_PREC_BF16_TC, fuse=1)
    if u8:
        net.predict_image_u8(x)
    else:
        net.predict(x)
    return net


def _assert_bit_equal(ref, got, what):
    """got: fused; ref: unfused.  Only the stem output is missing from the fused run."""
    for i in range(ref.n):
        r, g = util.fetched(ref, i), util.fetched(got, i)
        if i == 0:
            assert r is not None and g is None, what
            continue
        assert (r is None) == (g is None), (what, i)
        if r is not None:
            assert np.array_equal(r, g), (what, i)
    dr, dg = ref.detection_outputs(), got.detection_outputs()
    assert dr.keys() == dg.keys() and dr
    for i in dr:
        assert np.array_equal(dr[i], dg[i]), (what, "det", i)


@pytest.mark.parametrize("name,hw,batch", CASES)
def test_stem_s2_fused_bit_equal_to_unfused(name, hw, batch, workdir, monkeypatch):
    cfg, wts = _files_for(workdir, name, hw)
    x = cfgs.synthetic_images(batch, 3, hw[0], hw[1], seed=61)
    ref = _run(cfg, wts, batch, x, monkeypatch, fused=False)
    got = _run(cfg, wts, batch, x, monkeypatch, fused=True)
    _assert_bit_equal(ref, got, (name, hw, batch))


def test_stem_s2_u8_frames_bit_equal(workdir, monkeypatch):
    hw, batch = (96, 160), 3
    cfg, wts = _files_for(workdir, "s2chain", hw)
    frames = np.random.default_rng(62).integers(0, 256, (batch, hw[0], hw[1], 3), dtype=np.uint8)
    ref = _run(cfg, wts, batch, frames, monkeypatch, fused=False, u8=True)
    got = _run(cfg, wts, batch, frames, monkeypatch, fused=True, u8=True)
    _assert_bit_equal(ref, got, "u8")


def test_stem_s2_yolov3_608_bit_equal(workdir, monkeypatch):
    secs = cfgs.MODELS["yolov3"](608, 608)
    cfg, wts = util.write_net(workdir, "stems2_yolov3_608", secs, 1)
    x = cfgs.synthetic_images(2, 3, 608, 608, seed=63)
    ref = _run(cfg, wts, 2, x, monkeypatch, fused=False)
    got = _run(cfg, wts, 2, x, monkeypatch, fused=True)
    _assert_bit_equal(ref, got, "yolov3-608")


def test_stem_s2_layer1_vs_oracle(workdir, monkeypatch):
    from oracle import port
    hw, batch = (232, 136), 3
    cfg, wts = _files_for(workdir, "s2chain", hw)
    x = cfgs.synthetic_images(batch, 3, hw[0], hw[1], seed=64)
    net = _run(cfg, wts, batch, x, monkeypatch, fused=True)
    l0, l1 = net.layers[0], net.layers[1]
    stem = bf16_round(port.conv_fp32(bf16_round(x), bf16_round(l0["weights"]), l0["biases"], l0["n"], 3, 1, 1, l0["activation"]))
    exp = bf16_round(port.conv_fp32(stem, bf16_round(l1["weights"]), l1["biases"], l1["n"], 3, 2, 1, l1["activation"]))
    err = util.rel_l2(net.fetch_layer(1), exp)
    assert err <= 5e-4, err


def test_stem_s2_small_grids_bit_equal(workdir, monkeypatch):
    """1, 2 and 3 persistent CTAs walk many tiles each (partial tiles included)."""
    hw, batch = (80, 48), 5
    cfg, wts = _files_for(workdir, "s2chain", hw)
    x = cfgs.synthetic_images(batch, 3, hw[0], hw[1], seed=65)
    monkeypatch.delenv("YB_TC_GRID", raising=False)
    full = _run(cfg, wts, batch, x, monkeypatch, fused=True)
    for grid in ("1", "2", "3"):
        monkeypatch.setenv("YB_TC_GRID", grid)
        net = _run(cfg, wts, batch, x, monkeypatch, fused=True)
        for i in range(1, net.n):
            r, g = util.fetched(full, i), util.fetched(net, i)
            assert (r is None) == (g is None), (grid, i)
            if r is not None:
                assert np.array_equal(r, g), (grid, i)
        for i, o in full.detection_outputs().items():
            assert np.array_equal(o, net.detection_outputs()[i]), (grid, "det", i)


def test_stem_s2_engine_behaviour(workdir, monkeypatch):
    import yolo2_light_b200 as yb
    hw, batch = (64, 64), 2
    cfg, wts = _files_for(workdir, "s2chain", hw)
    x = cfgs.synthetic_images(batch, 3, hw[0], hw[1], seed=66)
    ref = _run(cfg, wts, batch, x, monkeypatch, fused=False)
    got = _run(cfg, wts, batch, x, monkeypatch, fused=True)
    with pytest.raises(yb.YbError):
        got.fetch_layer(0)
    assert got.last_launches() == ref.last_launches() - 1
    prof = got.profile()
    assert [k for li, k, _ in prof if li == 1] == ["conv_tc"], prof
    assert not [k for li, k, _ in prof if li == 0], prof
    # with fusion off (fuse = 0) the stem runs on its own and layer 0 stays readable
    monkeypatch.delenv("YB_NO_STEM_S2_FUSE", raising=False)
    net = util.load(cfg, wts, batch, fuse=0)
    net.predict(x)
    assert net.fetch_layer(0).shape[1] == 32
