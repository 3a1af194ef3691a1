"""The tensor-core convolutions bit for bit, on data on which they are exact (exact_model): every output is known to the
bit, so a single wrong element -- a stale ring stage, a wrong bias column, a tile row stored in the wrong place -- fails the
comparison, where a rel-L2 bound over the tensor would not notice it.

A layer under test that writes bf16 needs a consumer (a convolution without one writes f32): a one-hot 3x3 convolution
(bias 0, linear, one weight of 1 per filter) whose filters see the tested output through every tap, border included.  Its
output is a set of exactly shifted copies of the tested output, so a value stored into a zero border or into a pad row of a
merged-row tile shows up bitwise.  Each case names the edge of the tile planner it is for and asserts it through
Network.tc_plan.

The "tf32_" cases run the same edges under the GPU INT8 rule (`quantized` = 2), where every float convolution with a reader
runs on the tf32 wgmma of k_conv_tc and stores f32.  Their consumers read the tested output as tf32 operands: the expected
copies are exact_model.tf32_round of it, in the one conversion mode the whole output shows.

The helpers and the case table run on the CPU; the tests that need a GPU are marked."""
import numpy as np
import pytest

import exact_model
import ybtest_util as util
from exact_model import (BOUND_UNITS, F32_01, LEAKY, LINEAR, LOGISTIC, RELU, Net, conv_acc, epilogue, grid_acts, grid_bias,
                         grid_step, grid_weights, leaky_exact, leaky_tc, onehot, premise, run_reference, shifted_copies,
                         tf32_round)
from yolo2_light_b200 import cfgs


# ---- the case table -----------------------------------------------------------------------------------------------------
def c_bk(C, bk, rule=0):
    n = Net(C, 9, 11, 2, 100 + C, rule=rule)
    i = n.conv(64)
    n.consume()
    return n.edge(i, f"BK {bk} at C = {C}", lambda p: p["BK"] == bk)


def c_filters(nf, bn=None, rule=0):
    n = Net(32, 7, 5, 3, 200 + nf, rule=rule)
    i = n.conv(nf)
    n.consume()
    if bn:
        n.env["YB_TC_BN"] = str(bn)
    n.edge(i, f"n = {nf} not a multiple of BN", lambda p: nf % p["BN"] != 0 and p["nt"] == -(-nf // p["BN"]))
    if bn or (rule == 2 and nf > 128):   # k_conv_tc: at most 128 filters per tile
        n.edge(i, "two or more filter tiles", lambda p: p["nt"] >= 2)
    if rule == 2 and nf <= 32:
        n.edge(i, "BN 32: the second warpgroup idles in the epilogue", lambda p: p["BN"] == 32)
    return n


def c_f32(nf, size=3, stats=False):
    n = Net(64, 13, 7, 2, 300 + nf)
    i = n.conv(nf, size, act=LEAKY if nf != 255 else LINEAR, kern="tc")
    if stats:
        n.env["YB_TC_STATS"] = "1"
    return n.edge(i, f"f32 output, n = {nf}", lambda p: p["kernel"] == "k_conv_tc" and p["kind"] == "bf16")


def c_width(h, w, rule=0):
    n = Net(32, h, w, 3, 400 + 7 * h + w, rule=rule)
    i = n.conv(64)
    n.consume()
    return n.edge(i, f"OW {w} < TW, OW % TW != 0, or one-pixel tiles",
                  lambda p: w < p["TW"] or w % p["TW"] != 0 or p["TW"] == w == 1)


def c_tw128(w, batch, rule=0):
    n = Net(16, 1, w, batch, 500 + w, rule=rule)
    i = n.conv(32)
    n.consume()
    return n.edge(i, "TW = 128: a k_conv_tc_reg half tile is half a pixel row", lambda p: p["TW"] == 128)


def c_many_images_s1(rule=0):
    n = Net(32, 2, 2, 33, 601, rule=rule)
    i = n.conv(32)
    n.consume()
    return n.edge(i, "one tile spans 8+ images (stride 1: 4 merged rows each)", lambda p: p["TH"] >= 8 * 4)


def c_many_images_s2(rule=0):
    n = Net(32, 4, 6, 17, 602, rule=rule)
    i = n.conv(64, 3, 2)
    n.consume()
    return n.edge(i, "one tile spans 3+ images (stride 2: 3 merged half rows each)", lambda p: p["TH"] >= 3 * 3)


def c_straddle(h, w, batch, rule=0):
    n = Net(32, h, w, batch, 700 + h + w, rule=rule)
    i = n.conv(64, 3, 2)
    n.consume()
    # merged half rows: OH + 1 per image; a half tile of TH / 2 rows straddles two images unless it divides them
    return n.edge(i, "stride-2 half tiles straddle images",
                  lambda p: max(p["TH"] // 2, 1) > 1 and (h // 2 + 1) % max(p["TH"] // 2, 1) != 0)


def c_bump():
    n = Net(32, 30, 2, 5, 801)
    i = n.conv(32, 3, 2)
    n.consume()
    n.env["YB_TC_BN"] = "32"
    return n.edge(i, "stride 2, BN 32: TW 1 -> 2", lambda p: p["BN"] == 32 and p["TW"] == 2)


def c_knobs(bn=None, no_bstat=False, grid=None, stride=1, stats=False, rule=0, c=64, nf=256, batch=2):
    """rule 2: k_conv_tc takes its filter tile width from n alone (YB_TC_BN is k_conv_tc_reg's), so nf picks BN"""
    n = Net(c, 12, 10, batch, 900 + (bn or 0) + 7 * (grid or 0) + stride + 3 * stats, rule=rule)
    i = n.conv(nf, 3, stride)
    n.consume()
    if bn:
        if rule == 0:
            n.env["YB_TC_BN"] = str(bn)
        n.edge(i, f"BN {bn}", lambda p: p["BN"] == bn)
    if no_bstat:
        n.env["YB_TC_NO_BSTAT"] = "1"
        n.edge(i, "filter tiles streamed", lambda p: p["bstat"] == 0)
    if grid:
        n.env["YB_TC_GRID"] = str(grid)
        n.edge(i, f"{grid} CTAs, several work items each", lambda p: p["grid"] == grid and p["num_work"] > grid)
    if stats:   # the role-counter instantiations compute the same bits
        n.env["YB_TC_STATS"] = "1"
    return n


def c_shortcut(act2, fuse, rule=0):
    """rule 2: the fused conv + shortcut runs on the CUDA cores (f32 in, out and residual); unfused, the conv runs on tf32
    and k_shortcut adds the residual"""
    n = Net(64, 10, 6, 3, 1000 + fuse + (act2 == LEAKY), rule=rule)
    n.preserve()
    i = n.conv(64, kern="simt" if rule == 2 and fuse else None)
    n.add("shortcut", **{"from": "-2", "activation": act2})
    n.consume()
    n.fuse = fuse
    if rule == 2:
        return n.edge(i, f"shortcut act2 {act2}, fuse 0", lambda p: p["kind"] == "tf32") if not fuse else n
    return n.edge(i, f"shortcut act2 {act2}, fuse {fuse}", lambda p: p["kernel"] == "k_conv_tc_reg")


def c_concat(first, rule=0):
    """two tested layers write channel slices of one [route] buffer, each beside the other"""
    n = Net(32, 8, 6, 2, 1100 + first, rule=rule)
    n.preserve()
    a = n.conv(40)                        # 1
    n.add("route", layers="-2")           # 2: alias of layer 0
    b = n.conv(24)                        # 3
    n.add("route", layers="-3, -1" if first else "-1, -3")
    n.consume()
    pos = "first" if first else "second"
    # a channel slice: the output's pixel stride is the concat's 64 channels, not the layer's own
    kern = "k_conv_tc" if rule == 2 else "k_conv_tc_reg"
    n.edge(a, f"layer 1 writes the {pos} slice", lambda p: p["kernel"] == kern and p["out_ldc"] == 64)
    return n.edge(b, "layer 3 writes the other slice", lambda p: p["kernel"] == kern and p["out_ldc"] == 64)


def c_slice_input():
    """rule 2: a tf32 layer reads a channel slice of a [route] buffer through a single-input route: its input's pixel
    stride is the concat's 64 channels, its own channels the slice's 40"""
    n = Net(32, 8, 6, 2, 1150, rule=2)
    n.preserve()
    # 1: a one-hot 1x1 selection, linear, grid bias: layer 6 reads values on the activation grid
    n.conv(40, 1, 1, LINEAR, w=onehot(40, 32, 1, [(int(c), 0) for c in n.rng.integers(0, 32, 40)]), b=grid_acts(n.rng, 40, 8, -4, 4))
    n.add("route", layers="-2")               # 2: alias of layer 0
    n.conv(24)                                # 3
    n.add("route", layers="-3, -1")           # 4: [layer 1, layer 3]
    n.add("route", layers="-4")               # 5: alias of layer 1, a slice of layer 4's buffer
    i = n.conv(32)                            # 6
    n.consume()
    return n.edge(1, "layer 1 writes the first slice", lambda p: p["out_ldc"] == 64).edge(i, "C = 40: BK 8", lambda p: p["BK"] == 8)


def c_yolo(rule):
    """rule 1: the tf32 head of an INT8 network (parsed quantized); rule 2: parsed without INT8 layers"""
    n = Net(64, 6, 10, 2, 1200 + rule, calib=[16] * 4 if rule == 1 else None, rule=rule)
    i = n.conv(255, 1, act=LINEAR, kern="tc")
    n.secs.append(cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9))
    n.quantized = int(rule == 1)
    kind = "tf32" if rule else "bf16"
    return n.edge(i, f"fused [yolo], {kind}", lambda p: p["kind"] == kind and p["kernel"] == "k_conv_tc")


def c_refused(size):
    n = Net(8, 6, 10, 2, 1300 + size)
    n.conv(16, size, 2 if size == 1 else 1, kern="simt")
    n.consume()
    return n


def c_odd_s2():
    """rule 2: a stride-2 layer on an odd-sized input, which the tile's (half, parity) view cannot express: the CUDA cores"""
    n = Net(32, 7, 9, 2, 1350, rule=2)
    n.conv(64, 3, 2, kern="simt")
    n.consume()
    return n


def c_tf32_into_s8():
    """parsed quantized = 1, run under rule 2: a tf32 1x1 layer (index 0: float) feeds an INT8 3x3 layer; the INT8 layer is
    checked against the GPU rule's oracle on the tf32 layer's fetched output"""
    n = Net(32, 9, 7, 3, 1360, calib=[16] * 4, rule=2)
    i = n.conv(32, 1)
    j = n.conv(40, kern="s8_gpu")
    n.quantized = 1
    return n.edge(i, "tf32 1x1 into INT8", lambda p: p["kind"] == "tf32").edge(j, "s8_gpu", lambda p: p["kind"] == "s8_gpu")


def c_simt_shortcut():
    """12 filters: no whole 16-byte bf16 filter groups, so the CUDA cores run the layer, with the shortcut behind it fused
    (k_conv_simt<SimtF32<bf16, bf16, bf16>>: bf16 input, output and residual)"""
    n = Net(12, 7, 9, 3, 1700)
    n.preserve(kern="simt")
    i = n.conv(12, kern="simt")
    n.add("shortcut", **{"from": "-2", "activation": LEAKY})
    n.consume()
    return n


def c_simt_act(act):
    """relu and logistic, which the tensor cores refuse; the consumer copies the logistic's bf16 values, so it inherits
    their one-ulp tolerance"""
    n = Net(16, 6, 10, 2, 1800 + len(act))
    i = n.conv(16, act=act, kern="simt")
    j = n.consume()
    if act == LOGISTIC:
        n.tol = {i: 1, j: 1}
    return n


def c_simt_n4():
    n = Net(16, 7, 5, 3, 1900)
    n.conv(4, kern="simt")
    n.consume()
    return n


def c_stem(nf, h, w, batch):
    n = Net(3, h, w, batch, 1400 + nf + h)
    i = n.conv(nf, kern="stem", w=(n.rng.integers(-8, 9, (nf, 3, 3, 3)) / 64).astype(np.float32))
    n.consume()
    n.env["YB_NO_STEM_S2_FUSE"] = "1"
    return n.edge(i, f"k_stem_tc, n = {nf}", lambda p: p["kernel"] == "k_stem_tc")


def c_stem_s2(h, w, batch):
    n = Net(3, h, w, batch, 1500 + h + w)
    # linear stem, small weights: its bf16 output (layer 1's input) stays on a grid fine enough for the bound
    n.conv(32, act=LINEAR, kern="stem_s2", w=(n.rng.integers(-2, 3, (32, 3, 3, 3)) / 64).astype(np.float32),
           b=grid_bias(n.rng, 32, 512, 64))
    i = n.conv(64, 3, 2, kern="stem_s2", w=(n.rng.integers(-2, 3, (64, 32, 3, 3)) / 64).astype(np.float32))
    n.consume()
    return n.edge(i, "k_stem_s2_tc: stem + layer 1", lambda p: p["kernel"] == "k_stem_s2_tc")


def c_calibration(rule=0):
    """the largest K (3x3x1024) at the largest sums: images of 7/8 and 1 (on the 1/8 grid), a filter of +1/8 weights and one
    of -1/8 weights: |sum| ~ 1080 = 2^19.08 units of the 2^-9 product grid at every interior pixel; the other filters mix
    large and small addends.  f32 output: the accumulator itself, not rounded to bf16.  Rule 2: the same sums on the tf32
    wgmma, read by a [route] alias (a convolution without a reader runs on the CUDA cores)."""
    n = Net(1024, 5, 5, 2, 1600, rule=rule)
    w = grid_weights(n.rng, 32, 1024, 3)
    w[0] = 8 / 64
    w[1] = -8 / 64
    w[2] = np.where(n.rng.random((1024, 3, 3)) < 0.5, 8 / 64, 1 / 64)
    i = n.conv(32, act=LINEAR, kern="tc", w=w)
    n.x = (n.rng.integers(7, 9, (2, 1024, 5, 5)) / 8).astype(np.float32)
    if rule == 2:
        n.add("route", layers="-1")
    return n.edge(i, "K = 9216 at 2^19 product-grid units", lambda p: p["BK"] == (32 if rule == 2 else 64))


CASES = {
    "calibration": c_calibration,
    **{f"bk{bk}_c{C}": (lambda C=C, bk=bk: c_bk(C, bk)) for C, bk in [(16, 16), (48, 16), (80, 16), (112, 16), (96, 32),
                                                                       (32, 32), (192, 64)]},
    **{f"n{nf}": (lambda nf=nf: c_filters(nf)) for nf in (8, 24, 40, 72, 136, 264)},
    "n520_bn128": lambda: c_filters(520, 128),
    "n136_bn64": lambda: c_filters(136, 64),
    **{f"f32_n{nf}": (lambda nf=nf: c_f32(nf, 1 if nf == 255 else 3)) for nf in (9, 18, 75, 255)},
    **{f"w{w}_h{h}": (lambda h=h, w=w: c_width(h, w)) for h, w in [(5, 1), (3, 3), (9, 7), (11, 13), (7, 19), (3, 37)]},
    "tw128_w256": lambda: c_tw128(256, 1),
    "tw128_w200_b3": lambda: c_tw128(200, 3),
    "images_s1_b33": c_many_images_s1,
    "images_s2_b17": c_many_images_s2,
    "straddle_6x10": lambda: c_straddle(6, 10, 3),
    "straddle_38x38": lambda: c_straddle(38, 38, 3),
    "s2_bn32_tw_bump": c_bump,
    **{f"bn{bn}": (lambda bn=bn: c_knobs(bn=bn)) for bn in (32, 64, 128, 256)},
    "bn64_s2": lambda: c_knobs(bn=64, stride=2),
    "streamed": lambda: c_knobs(bn=64, no_bstat=True),
    "streamed_s2": lambda: c_knobs(bn=128, no_bstat=True, stride=2),
    "grid1": lambda: c_knobs(grid=1),
    "grid3": lambda: c_knobs(bn=32, grid=3),
    "grid3_s2": lambda: c_knobs(bn=64, grid=3, stride=2),
    "stats_grid3": lambda: c_knobs(bn=128, grid=3, stats=True),
    "stats_grid3_s2": lambda: c_knobs(bn=64, grid=3, stride=2, stats=True),
    "stats_f32_n75": lambda: c_f32(75, stats=True),
    **{f"shortcut_{a}_fuse{f}": (lambda a=a, f=f: c_shortcut(a, f)) for a in (LINEAR, LEAKY) for f in (0, 1)},
    "concat_first": lambda: c_concat(True),
    "concat_second": lambda: c_concat(False),
    "yolo_bf16": lambda: c_yolo(0),
    "yolo_tf32": lambda: c_yolo(1),
    "refused_c8_1x1s2": lambda: c_refused(1),
    "refused_c8_3x3": lambda: c_refused(3),
    "simt_n12_shortcut": c_simt_shortcut,
    "simt_relu": lambda: c_simt_act(RELU),
    "simt_logistic": lambda: c_simt_act(LOGISTIC),
    "simt_n4": c_simt_n4,
    "stem16": lambda: c_stem(16, 10, 14, 3),
    "stem32": lambda: c_stem(32, 7, 9, 2),
    **{f"stem_s2_{h}x{w}_b{b}": (lambda h=h, w=w, b=b: c_stem_s2(h, w, b)) for h, w, b in [(16, 16, 2), (38, 22, 3), (64, 48, 1)]},
    # the GPU INT8 rule's float layers: k_conv_tc on the tf32 wgmma, f32 out.  BK 8 / 16 / 32: 1, 2, 4 wgmmas per K-block
    "tf32_calibration": lambda: c_calibration(2),
    **{f"tf32_bk{bk}_c{C}": (lambda C=C, bk=bk: c_bk(C, bk, 2)) for C, bk in [(8, 8), (24, 8), (40, 8), (16, 16), (48, 16),
                                                                             (80, 16), (32, 32), (96, 32)]},
    **{f"tf32_n{nf}": (lambda nf=nf: c_filters(nf, rule=2)) for nf in (8, 9, 24, 40, 72, 75, 136, 264)},
    **{f"tf32_w{w}_h{h}": (lambda h=h, w=w: c_width(h, w, 2)) for h, w in [(5, 1), (3, 3), (9, 7), (11, 13), (7, 19), (3, 37)]},
    "tf32_tw128_w256": lambda: c_tw128(256, 1, 2),
    "tf32_tw128_w200_b3": lambda: c_tw128(200, 3, 2),
    "tf32_images_s1_b33": lambda: c_many_images_s1(2),
    "tf32_images_s2_b17": lambda: c_many_images_s2(2),
    "tf32_straddle_6x10": lambda: c_straddle(6, 10, 3, 2),
    "tf32_straddle_38x38": lambda: c_straddle(38, 38, 3, 2),
    "tf32_odd_s2": c_odd_s2,
    **{f"tf32_s2_bn{bn}": (lambda bn=bn, nf=nf: c_knobs(bn=bn, stride=2, rule=2, nf=nf)) for bn, nf in [(32, 24), (64, 40), (128, 136)]},
    "tf32_streamed": lambda: c_knobs(no_bstat=True, rule=2, c=16, nf=24),
    "tf32_streamed_s2": lambda: c_knobs(no_bstat=True, stride=2, rule=2, c=16, nf=40),
    "tf32_grid1": lambda: c_knobs(grid=1, rule=2, nf=72),
    "tf32_grid3": lambda: c_knobs(grid=3, rule=2, nf=136),
    "tf32_grid3_s2": lambda: c_knobs(grid=3, stride=2, rule=2, nf=136, batch=8),
    "tf32_stats_grid3": lambda: c_knobs(grid=3, stats=True, rule=2, nf=136),
    "tf32_stats_grid3_s2": lambda: c_knobs(grid=3, stride=2, stats=True, rule=2, nf=136, batch=8),
    **{f"tf32_shortcut_{a}_fuse{f}": (lambda a=a, f=f: c_shortcut(a, f, 2)) for a in (LINEAR, LEAKY) for f in (0, 1)},
    "tf32_concat_first": lambda: c_concat(True, 2),
    "tf32_concat_second": lambda: c_concat(False, 2),
    "tf32_slice_input": c_slice_input,
    "tf32_yolo": lambda: c_yolo(2),
    "tf32_into_s8_gpu": c_tf32_into_s8,
}


def build_case(name):
    net = CASES[name]()
    if net.x is not None:
        return net, net.x
    stem = net.kern.get(0, "").startswith("stem")
    x = net.images(16, 0, 16) if stem else net.images()
    return net, x


# ---- CPU tests ----------------------------------------------------------------------------------------------------------
def test_calibration_case_reaches_the_top_of_the_bound():
    """the calibration cases (bf16 and tf32) hold the accumulator between 2^19 and 2^20 units of its product grid (2^-9)"""
    for name in ("calibration", "tf32_calibration"):
        net, x = build_case(name)
        w, b = net.params[0]
        assert grid_step(x) * grid_step(w) == 2.0 ** -9 and grid_step(b) >= 2.0 ** -9
        _, units = run_reference(net, x, adt_bf16=not net.rule)
        assert 2 ** 19 <= units[0] < BOUND_UNITS, (name, units[0])


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_premise(name):
    """every convolution of every case is exact on the tensor cores: on the grid and below 2^20 product-grid units"""
    net, x = build_case(name)
    _, units = run_reference(net, x, adt_bf16=not net.rule)
    assert units and max(units.values()) < BOUND_UNITS


@pytest.mark.parametrize("shape", [(16, 5, 7, 24, 3, 1, 2), (48, 6, 4, 40, 3, 2, 3), (64, 3, 9, 9, 1, 1, 2),
                                   (192, 4, 4, 32, 3, 1, 1), (32, 1, 37, 72, 3, 1, 3)])
def test_reference_equals_oracle_on_grid_data(shape):
    """float64 per-tap matmul + the f32 epilogue == the oracle's f32 convolution (which sums in k order -- also exact on grid
    data), bit for bit, linear activation"""
    from oracle import port
    C, H, W, n, k, s, B = shape
    rng = np.random.default_rng(C + H + n)
    x = grid_acts(rng, (B, C, H, W))
    w = grid_weights(rng, n, C, k)
    b = grid_bias(rng, n)
    premise(x.transpose(0, 2, 3, 1), w, b, s, k // 2)
    ref = epilogue(conv_acc(x.transpose(0, 2, 3, 1), w, s, k // 2), b, LINEAR, "reg", bf16=False)
    exp = port.conv_fp32(x, w, b, n, k, s, k // 2, 3)
    assert util.bits_equal(ref.transpose(0, 3, 1, 2), exp)


def test_leaky_emulations_differ_where_the_kernels_do():
    """fmaxf(a, 0.1f a) and (float)(0.1 (double) a) are different functions: the two epilogue emulations are not
    interchangeable"""
    a = -(np.arange(1, 4097, dtype=np.float32) / 512)
    assert not np.array_equal(leaky_tc(a), leaky_exact(a))


def _tested_layers(net):
    """the float layers the cases test (an INT8 layer is checked against the oracle instead)"""
    one_hot = lambda w: np.all((w != 0).reshape(len(w), -1).sum(1) <= 1)
    return [i for i, (w, _) in net.params.items() if not one_hot(w) and net.kern[i] != "s8_gpu"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_sensitivity(name):
    """a kernel that skips a K-block or misindexes a bias cannot pass by luck: dropping any single (tap, channel group) of
    a tested layer's weights -- 16 channels, 8 under rule 2, the narrowest K-block of each kind -- or moving one filter's
    bias by one grid step, changes at least one expected output"""
    net, x = build_case(name)
    outs, _ = run_reference(net, x, adt_bf16=not net.rule)
    group = 8 if net.rule == 2 else 16
    shapes = net.shapes()
    for i in _tested_layers(net):
        L = shapes[i]
        cur = np.ascontiguousarray(x.transpose(0, 2, 3, 1)) if i == 0 else outs[i - 1]
        if net.kern[i].startswith("stem") and i == 0:
            cur = util.bf16_round(cur)
        w, b = net.params[i]
        bf16 = not net.rule and shapes[i + 1]["type"] != "yolo" if i + 1 < len(shapes) else False
        act = L["activation"]
        base = epilogue(conv_acc(cur, w, L["stride"], L["pad"]), b, act, net.kern[i], bf16=bf16)
        C, k = w.shape[1], w.shape[2]
        for t in range(k * k):
            for g in range(0, C, group):
                w2 = w.copy()
                w2[:, g:g + group, t // k, t % k] = 0
                if not np.any(conv_acc(cur, w - w2, L["stride"], L["pad"])):
                    continue   # nothing to drop: zero weights, or a tap that only ever reads the zero border
                e = epilogue(conv_acc(cur, w2, L["stride"], L["pad"]), b, act, net.kern[i], bf16=bf16)
                assert not np.array_equal(e, base), (name, i, "tap", t, "channels", g)
        acc = conv_acc(cur, w, L["stride"], L["pad"])
        for f in range(len(b)):
            b2 = b.copy()
            b2[f] += np.float32(1 / 512)
            e = epilogue(acc[..., f:f + 1], b2[f:f + 1], act, net.kern[i], bf16=bf16)
            assert not np.array_equal(e, base[..., f:f + 1]), (name, i, "bias", f)


# ---- GPU tests ----------------------------------------------------------------------------------------------------------
KERNEL_OF = {"reg": "k_conv_tc_reg", "tc": "k_conv_tc", "stem": "k_stem_tc", "stem_s2": "k_stem_s2_tc", "s8_gpu": "k_conv_tc"}
TF32_MODES = ("rz", "rn", "rna")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_tc_exact(name, workdir, monkeypatch):
    net, x = build_case(name)
    exp, _ = run_reference(net, x, adt_bf16=not net.rule)
    for k, v in net.env.items():
        monkeypatch.setenv(k, v)
    m = util.load(*exact_model.write_net(net, workdir, name), net.batch, quantized=net.quantized, fuse=net.fuse)
    q = net.rule
    # the plan of every convolution is the one the case is for
    for i, kern in net.kern.items():
        p = m.tc_plan(i, quantized=q)
        if kern == "simt":
            assert p == {}, (name, i, p)
        else:
            assert p.get("kernel") == KERNEL_OF[kern], (name, i, p)
            if q == 2:
                assert p["kind"] == ("s8_gpu" if kern == "s8_gpu" else "tf32"), (name, i, p)
    for i, what, pred in net.edges:
        p = m.tc_plan(i, quantized=q)
        assert pred(p), (name, what, p)
    # the CUDA-core layers: one k_conv_simt launch each, the bf16 instantiation in a bf16 network, and no launch for a
    # shortcut fused into one
    # (the last layer's NCHW copy, k_nhwc_to_nchw_f32, is an op of that layer too)
    ops = [op for op in m.op_kernels(quantized=q) if op[2] is None or "k_nhwc_to_nchw_f32" not in op[2]]
    shapes = net.shapes()
    for i, kern in net.kern.items():
        if kern != "simt":
            continue
        mine = [k for j, _, k in ops if j == i]
        assert len(mine) == 1 and "k_conv_simt" in mine[0] and "SimtF32" in mine[0], (name, i, mine)
        assert ("__nv_bfloat16" in mine[0]) == (not q), (name, i, mine)
        if i + 1 < len(shapes) and shapes[i + 1]["type"] == "shortcut" and net.fuse and shapes[i]["stride"] == 1:
            assert not [k for j, _, k in ops if j == i + 1], (name, i + 1, ops)
    m.predict(x, quantized=q)
    # the one-hot consumer and what reads it: checked against shifted copies below (on tf32 they are not run_reference's)
    last = max(i for i, L in enumerate(shapes) if L["type"] == "convolutional")
    consumer = last if net.params[last][0].shape[2] == 3 and _is_consumer(net, last) else None
    checked = 0
    for i, L in enumerate(shapes):
        if net.kern.get(i) == "s8_gpu":   # the INT8 layer against the GPU rule's oracle on its fetched input
            e, _ = util.oracle_layer(m.layers[i], i, m.fetch_layer(i - 1, quantized=q), q)
            assert util.bits_equal(m.fetch_layer(i, quantized=q), e), (name, i)
            checked += 1
            continue
        if consumer is not None and i >= consumer and net.kern[consumer] == "tc" and q == 2:
            continue
        e = exp.get(i)
        if L["type"] == "yolo":
            got = m.detection_outputs()[i]
            v = exp[i - 1].transpose(0, 3, 1, 2)        # head values, NCHW
            per = 4 + 80 + 1
            raw = np.isin(np.arange(v.shape[1]) % per, (2, 3))
            assert util.bits_equal(got[:, raw], v[:, raw]), name
            sg = 1.0 / (1.0 + np.exp(-v[:, ~raw].astype(np.float64)))
            err = np.abs(got[:, ~raw] - sg) / sg
            assert np.all(err <= util.logistic_bound(v[:, ~raw])), (name, float(err.max()))
            checked += 1
            continue
        if e is None or (L["type"] == "convolutional" and i + 1 < len(shapes) and shapes[i + 1]["type"] == "yolo"):
            continue
        if net.kern.get(0) == "stem_s2" and i == 0:
            continue   # k_stem_s2_tc never writes the stem output
        got = m.fetch_layer(i, quantized=q).transpose(0, 2, 3, 1)
        assert got.shape == e.shape, (name, i)
        if net.tol.get(i):
            d = util.ulp_diff(got, e, True)
            assert np.all(got >= 0) and np.all(e >= 0) and np.array_equal(np.signbit(got), np.signbit(e)) and \
                d.max() <= net.tol[i], (name, i, int(d.max()))   # logistic > 0, border 0
            checked += 1
            continue
        bad = np.argwhere(got.view(np.uint32) != np.ascontiguousarray(e).view(np.uint32))
        assert len(bad) == 0, (name, i, len(bad), bad[:5].tolist())
        checked += 1
    if consumer is not None:
        # the consumer against shifted copies of its input, computed independently of run_reference: every tap that reads
        # the border gives +0, so a value stored into a border or a pad row fails here
        pairs = [(int(c), int(ky * 3 + kx)) for _, c, ky, kx in np.argwhere(net.params[consumer][0] == 1)]   # ordered by filter
        src = m.fetch_layer(consumer - 1, quantized=q).transpose(0, 2, 3, 1)
        got = m.fetch_layer(consumer, quantized=q).transpose(0, 2, 3, 1)
        if q == 2 and net.kern[consumer] == "tc":
            # tf32 operands: every element follows one conversion of f32 to tf32, and the modes differ on this input
            exps = {mode: shifted_copies(tf32_round(src, mode), pairs) for mode in TF32_MODES}
            assert not util.bits_equal(exps["rz"], exps["rn"]), name
            modes = [mode for mode in TF32_MODES if util.bits_equal(got, exps[mode])]
            bad = {mode: int(np.sum(got.view(np.uint32) != e.view(np.uint32))) for mode, e in exps.items()}
            assert modes, (name, "elements off each conversion mode", bad)
            print(name, "tf32 operand conversion:", modes)
            checked += 1
        else:
            assert util.bits_equal(got, shifted_copies(src, pairs)), name
    assert checked >= 1, name


def _is_consumer(net, i):
    w, b = net.params[i]
    return not np.any(b) and np.all((w != 0).reshape(len(w), -1).sum(1) == 1) and np.all(w[w != 0] == 1)


# ---- integer kinds at the edge shapes: bit for bit against the oracle on the fetched input ---------------------------
RULE_OF = {"s8": 1, "s8_gpu": 2, "xnor": 0}    # the INT8 rule each integer kind runs under


def _int_secs(C, h, w, quantized, calib=16):
    net = cfgs._net(w, h, [calib] * 8 if quantized else None)
    return [net, cfgs._conv(C, 3)]     # layer 0: f32 (the INT8 rule starts at layer 1), leaky


INT_SHAPES = [   # kind, C, n, h, w, stride, batch: padded channels (C % 32 != 0), n % 4 != 0, odd sizes, stride 2
    ("s8", 8, 8, 7, 9, 1, 3), ("s8", 24, 30, 9, 5, 1, 2), ("s8", 40, 40, 11, 13, 1, 1), ("s8", 100, 264, 5, 7, 1, 2),
    ("s8", 24, 30, 10, 14, 2, 3), ("s8", 40, 264, 6, 10, 2, 1), ("s8", 8, 40, 2, 2, 2, 5),
    ("xnor", 16, 8, 7, 9, 1, 3), ("xnor", 48, 40, 5, 3, 1, 2), ("xnor", 80, 264, 9, 11, 1, 1), ("xnor", 16, 30, 1, 13, 1, 3),
    ("s8_gpu", 8, 8, 7, 9, 1, 3), ("s8_gpu", 24, 30, 9, 5, 1, 2), ("s8_gpu", 40, 40, 11, 13, 1, 1),
    ("s8_gpu", 100, 264, 5, 7, 1, 2), ("s8_gpu", 24, 30, 10, 14, 2, 3), ("s8_gpu", 40, 264, 6, 10, 2, 1),
    ("s8_gpu", 8, 40, 2, 2, 2, 5),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,C,n,h,w,stride,batch", INT_SHAPES)
def test_integer_kinds_exact(kind, C, n, h, w, stride, batch, workdir):
    """s8_gpu: also with input multipliers of 2^20, where the GPU rule's conversion saturates at +-127"""
    import rule_oracle as ro
    q = RULE_OF[kind]
    for calib in (16, 2 ** 20) if q == 2 else (16,):
        secs = _int_secs(C, h, w, q, calib)
        secs.append(cfgs._conv(n, 3, stride, **({} if q else {"xnor": 1, "bin_output": 1})))
        name = f"int_{kind}_{C}_{n}_{h}x{w}s{stride}" + ("_sat" if calib != 16 else "")
        m = util.load(*util.write_net(workdir, name, secs, C + n), batch, quantized=int(q > 0))
        m.set_option("keep_counts", 1)
        p = m.tc_plan(1, quantized=q)
        assert p.get("kind") == kind and p["kernel"] == "k_conv_tc", p
        assert p["tma_epi"] == 0, p    # keep_counts: the raw accumulators go through the LSU stores
        m.predict(cfgs.synthetic_images(batch, 3, h, w, seed=C), quantized=q)
        x = m.fetch_layer(0, quantized=q)
        if calib != 16:
            xq = ro.quantize_input_gpu(x, m.layers[1]["input_quant_multipler"])
            assert np.any(xq == 127) and np.any(xq == -127), (x.min(), x.max())
        exp, acc = util.oracle_layer(m.layers[1], 1, x, q)
        assert np.array_equal(m.fetch_counts(1, quantized=q), acc)
        assert util.bits_equal(m.fetch_layer(1, quantized=q), exp)
        # and without the raw-accumulator dump: the TMA epilogue at stride 1, the LSU stores at stride 2
        m.set_option("keep_counts", 0)
        p = m.tc_plan(1, quantized=q)
        assert (p["tma_epi"] == 0) == (stride == 2), p
        m.predict(cfgs.synthetic_images(batch, 3, h, w, seed=C), quantized=q)
        assert util.bits_equal(m.fetch_layer(1, quantized=q), exp)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["s8", "xnor", "s8_gpu"])
def test_integer_kinds_role_counters(kind, workdir, monkeypatch, capfd):
    """YB_TC_STATS=1 runs the role-counter instantiation of the integer epilogue: the same bits as the oracle, and a TCSTATS
    line per plan when the network is freed"""
    import gc
    monkeypatch.setenv("YB_TC_STATS", "1")
    monkeypatch.setenv("YB_TC_GRID", "2")   # several work items per CTA
    q = RULE_OF[kind]
    secs = _int_secs(40 if q else 48, 11, 13, q) + [cfgs._conv(40, 3, **({} if q else {"xnor": 1, "bin_output": 1}))]
    m = util.load(*util.write_net(workdir, f"stats_{kind}", secs, 11), 2, quantized=int(q > 0))
    p = m.tc_plan(1, quantized=q)
    assert p.get("kind") == kind and p["kernel"] == "k_conv_tc" and p["num_work"] > p["grid"], p
    m.predict(cfgs.synthetic_images(2, 3, 11, 13, seed=4), quantized=q)
    exp, _ = util.oracle_layer(m.layers[1], 1, m.fetch_layer(0, quantized=q), q)
    assert util.bits_equal(m.fetch_layer(1, quantized=q), exp)
    capfd.readouterr()
    del m
    gc.collect()
    lines = [l for l in capfd.readouterr().err.splitlines() if l.startswith("TCSTATS")]
    assert lines and all("producer: wait_empty" in l and "consumers: wait_full" in l for l in lines), lines


@pytest.mark.gpu
@pytest.mark.parametrize("kind,h,w,batch", [("s8", 2, 2, 3), ("s8", 6, 10, 1), ("xnor", 2, 2, 3), ("xnor", 6, 10, 1),
                                            ("s8_gpu", 2, 2, 3), ("s8_gpu", 6, 10, 1)])
def test_pool_fused_epilogue_exact(kind, h, w, batch, workdir):
    """the 2x2/2 max-pool and the next layer's input conversion in the integer epilogue (s8, the GPU rule's saturating s8,
    +-1 bytes) at the smallest and odd-batch shapes it takes"""
    from oracle import port
    q = RULE_OF[kind]
    extra = {} if q else {"xnor": 1, "bin_output": 1}
    secs = _int_secs(32, h, w, q) + [cfgs._conv(32, 3, **extra), ("maxpool", {"size": "2", "stride": "2"}),
                                      cfgs._conv(32, 3, **extra)]
    m = util.load(*util.write_net(workdir, f"pool_{kind}_{h}x{w}", secs, 7 + h), batch, quantized=int(q > 0))
    p = m.tc_plan(1, quantized=q)
    assert p.get("kind") == kind and p["jshift"] == 1 and p["TW"] == 8, p    # pool fused: 8 x 16 tiles, one row down
    m.predict(cfgs.synthetic_images(batch, 3, h, w, seed=h), quantized=q)
    L = m.layers
    y1, _ = util.oracle_layer(L[1], 1, m.fetch_layer(0, quantized=q), q)
    y3, _ = util.oracle_layer(L[3], 3, port.maxpool(y1, L[2]["size"], L[2]["stride"], L[2]["pad"]), q)
    assert util.bits_equal(m.fetch_layer(3, quantized=q), y3)


@pytest.mark.gpu
def test_int8_slice_store_leaves_the_next_slice(workdir):
    """An INT8 stride-2 layer with n = 30 writes channels 0..29 of a [route] buffer whose channels 30.. belong to layer 1,
    which ran earlier (on the CUDA cores: its f32 slice is not 16-byte aligned).  The f32 LSU store of the tensor-core
    epilogue must stop at filter n, not at the next whole float4 group."""
    from oracle import port
    secs = _int_secs(16, 6, 10, True) + [cfgs._conv(16, 3),                       # 1: INT8, second slice
                                          ("upsample", {"stride": "2"}),            # 2
                                          cfgs._conv(30, 3, 2),                     # 3: INT8 stride 2, first slice
                                          ("route", {"layers": "-1, -3"}),          # 4: [layer 3, layer 1]
                                          cfgs._conv(16, 1)]
    m = util.load(*util.write_net(workdir, "slice_spill", secs, 5), 2, quantized=1)
    assert m.tc_plan(1, quantized=True) == {}
    p = m.tc_plan(3, quantized=True)
    assert p.get("kind") == "s8" and p["tma_epi"] == 0, p
    m.predict(cfgs.synthetic_images(2, 3, 6, 10, seed=3), quantized=True)
    L = m.layers
    y1, _ = util.oracle_layer(L[1], 1, m.fetch_layer(0, quantized=True), 1)
    y3, _ = util.oracle_layer(L[3], 3, port.upsample(y1, 2), 1)
    got = m.fetch_layer(4, quantized=True)
    assert util.bits_equal(got[:, :30], y3)
    assert util.bits_equal(got[:, 30:], y1), "layer 3 overwrote layer 1's channels"


# ---- production shapes: every distinct convolution of yolov3-608 and yolov3-spp-608 at batch 16, with its fusion ----------
def gpu_rule_floats(secs):
    """the convolutions a network parsed with quantized = 1 keeps float (l.quantized == 0): index 0, linear and 1x1 layers,
    stride-2 layers past index 1, and every convolution from the one whose second successor is a [yolo] layer on"""
    L = cfgs.conv_shapes(secs)
    floats, latched = [], False
    for i, l in enumerate(L):
        if l["type"] != "convolutional":
            continue
        latched |= i + 2 < len(L) and L[i + 2]["type"] == "yolo"
        if latched or i == 0 or l["activation"] == LINEAR or (i > 1 and l["stride"] > 1) or l["size"] == 1:
            floats.append(i)
    return floats


def production_shapes(rule=0, nets=None):
    """(C, H, W, n, size, stride, fusion) of every distinct convolution of the two networks at 608 x 608.  fusion: "stem_s2"
    (the stem and layer 1, one kernel), "shortcut" (3x3 + fused residual), "yolo" (head + fused [yolo]), "slice" (writes a
    channel slice of a [route] buffer) or "none".  rule 2: the float convolutions of the GPU INT8 rule but the stem, the
    layers that run on tf32."""
    keys = []
    for secs in nets or (cfgs.yolov3(608, 608), cfgs.yolov3_spp(608, 608)):
        L = cfgs.conv_shapes(secs)
        slices = {j for l in L if l["type"] == "route" and len(l["layers"]) > 1 for j in l["layers"]}
        tested = [i for i in gpu_rule_floats(secs) if i > 0] if rule == 2 else [i for i in range(len(L)) if i != 1]
        for i, l in enumerate(L):
            if l["type"] != "convolutional" or i not in tested:
                continue
            nxt = L[i + 1]["type"] if i + 1 < len(L) else None
            fusion = ("stem_s2" if i == 0 else "shortcut" if nxt == "shortcut" and l["stride"] == 1 else
                      "yolo" if nxt == "yolo" else "slice" if i in slices else "none")
            k = (l["c"], l["h"], l["w"], l["n"], l["size"], l["stride"], fusion)
            if k not in keys:
                keys.append(k)
    return keys


PRODUCTION = production_shapes()
PRODUCTION_TF32 = production_shapes(2)


def test_torch_reference_equals_numpy_reference():
    """the GPU-side float64 reference of the production shapes is the same function as conv_acc (run here on the CPU)"""
    import torch
    rng = np.random.default_rng(3)
    for C, n, k, s in ((32, 24, 3, 1), (48, 40, 3, 2), (64, 16, 1, 1)):
        x = grid_acts(rng, (2, 9, 7, C)).astype(np.float64)
        w = grid_weights(rng, n, C, k)
        got = _t_conv_acc(torch.as_tensor(x), w, s, k // 2).numpy()
        assert np.array_equal(got, conv_acc(x, w, s, k // 2))


def test_production_shapes_cover_both_networks():
    fusions = {k[-1] for k in PRODUCTION}
    assert fusions == {"stem_s2", "shortcut", "yolo", "slice", "none"}, fusions
    assert (1024, 19, 19, 512, 1, 1, "none") in PRODUCTION and (2048, 19, 19, 512, 1, 1, "none") in PRODUCTION


def test_production_tf32_shapes():
    """the GPU rule's tf32 layers: 19 distinct shapes in yolov3-608 (48 layers), two more in yolov3-spp-608 (the 1x1
    2048 -> 512 and the 1x1 that writes the SPP block's [route] slice); the four 3x3/2 downsampling layers among them"""
    v3 = cfgs.yolov3(608, 608)
    assert len(gpu_rule_floats(v3)) == 49 and len(production_shapes(2, [v3])) == 19
    assert len(PRODUCTION_TF32) == 21, len(PRODUCTION_TF32)
    assert {k[-1] for k in PRODUCTION_TF32} == {"none", "yolo", "slice"}
    assert [k for k in PRODUCTION_TF32 if k[5] == 2] == [(64, 304, 304, 128, 3, 2, "none"), (128, 152, 152, 256, 3, 2, "none"),
                                                         (256, 76, 76, 512, 3, 2, "none"), (512, 38, 38, 1024, 3, 2, "none")]
    assert (2048, 19, 19, 512, 1, 1, "none") in PRODUCTION_TF32 and (1024, 19, 19, 512, 1, 1, "slice") in PRODUCTION_TF32


def test_gpu_rule_floats_are_the_parsers():
    """gpu_rule_floats restates the parser's layer rule: the same float convolutions as yb.parse_network_cfg(quantized = 1)"""
    import tempfile
    import yolo2_light_b200 as yb
    d = tempfile.mkdtemp()
    for name, secs in (("v3", cfgs.yolov3(608, 608)), ("spp", cfgs.yolov3_spp(608, 608))):
        net = yb.parse_network_cfg(cfgs.write_cfg(secs, f"{d}/{name}.cfg"), 1, 1)
        assert gpu_rule_floats(secs) == [i for i, l in enumerate(net.layers)
                                         if l["type_name"] == "CONVOLUTIONAL" and not l["quantized"]], name


def production_net(key, batch=16, rule=0):
    """the single-layer case of one production shape, with the fusion the network uses there; returns (net, tested layer)"""
    C, H, W, n, k, s, fusion = key
    seed = C * 7 + n + H + k + s
    if fusion == "stem_s2":
        net = Net(3, H, W, batch, seed)
        net.conv(32, act=LINEAR, kern="stem_s2", w=(net.rng.integers(-2, 3, (32, 3, 3, 3)) / 64).astype(np.float32),
                 b=grid_bias(net.rng, 32, 512, 64))
        i = net.conv(64, 3, 2, kern="stem_s2", w=(net.rng.integers(-2, 3, (64, 32, 3, 3)) / 64).astype(np.float32))
        net.add("route", layers="-1")
        return net, i
    if fusion == "shortcut":
        # grid-preserving n -> n (the residual), a one-hot n -> C selection, the tested 3x3 C -> n, shortcut from layer 0
        net = Net(n, H, W, batch, seed)
        net.preserve()
        perm = net.rng.permutation(n)[:C]
        net.conv(C, 1, 1, LINEAR, w=onehot(C, n, 1, [(int(c), 0) for c in perm]), b=grid_acts(net.rng, C, 8, -4, 4))
        i = net.conv(n, k, s)
        net.add("shortcut", **{"from": "-3", "activation": LINEAR})
        net.add("route", layers="-1")
        return net, i
    net = Net(C, H, W, batch, seed, rule=rule)
    if fusion == "yolo":
        i = net.conv(n, k, s, act=LINEAR, kern="tc")
        net.secs.append(cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9))
        return net, i
    i = net.conv(n, k, s)
    if fusion == "slice":      # as in the SPP block: max-pools of the layer, concatenated with it
        net.add("maxpool", size=5, stride=1)
        net.add("route", layers="-1, -2")
    else:
        net.add("route", layers="-1")
    return net, i


def _t_conv_acc(x, w, stride, pad):
    """conv_acc with torch float64 on the GPU: exact on grid data in any summation order"""
    import torch
    B, H, W, C = x.shape
    n, _, k, _ = w.shape
    OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    xp = torch.nn.functional.pad(x, (0, 0, pad, pad, pad, pad))
    wt = torch.as_tensor(w, dtype=torch.float64, device=x.device)
    acc = torch.zeros((B, OH, OW, n), dtype=torch.float64, device=x.device)
    for ky in range(k):
        for kx in range(k):
            xs = xp[:, ky:ky + stride * (OH - 1) + 1:stride, kx:kx + stride * (OW - 1) + 1:stride, :]
            acc += xs @ wt[:, :, ky, kx].T
    return acc


def _t_grid_step(a):
    import torch
    for e in range(41):
        s = a * 2.0 ** e
        if bool(torch.equal(s, torch.round(s))):
            return 2.0 ** -e
    raise AssertionError("data off every binary grid")


def _t_layer(x, w, b, L, kern, res=None, act2=LINEAR, bf16=True):
    """premise and expected output of one convolution over NHWC float64 x on the GPU, as stored (float32)"""
    import torch
    nz = w != 0
    if not (np.all(nz.reshape(len(w), -1).sum(1) <= 1) and np.all(np.abs(w[nz]) == 1)):
        g = min(_t_grid_step(x) * grid_step(w), grid_step(b))
        units = float((_t_conv_acc(x.abs(), np.abs(w), L["stride"], L["pad"]).amax() + float(np.abs(b).max())) / g)
        assert units < BOUND_UNITS, units
    acc = _t_conv_acc(x, w, L["stride"], L["pad"])
    bt = torch.as_tensor(b, device=x.device)
    a = (acc + 0.0).float() + bt
    f01 = torch.tensor(F32_01, device=x.device)
    assert kern != "simt"
    if L["activation"] == LEAKY:
        a = torch.maximum(a, f01 * a)
    if res is not None:
        a = a + res
        if act2 == LEAKY:
            a = torch.maximum(a, f01 * a)
    return a.to(torch.bfloat16).float() if bf16 else a


def _t_bits_equal(got_nchw, exp_nhwc):
    import torch
    g = torch.as_tensor(np.ascontiguousarray(got_nchw), device=exp_nhwc.device).permute(0, 2, 3, 1)
    return g.shape == exp_nhwc.shape and bool(torch.equal(g.contiguous().view(torch.int32), exp_nhwc.contiguous().view(torch.int32)))


@pytest.mark.gpu
@pytest.mark.parametrize("key,rule", [pytest.param(k, 0, id="{}x{}x{}-n{}-k{}s{}-{}".format(*k)) for k in PRODUCTION] +
                         [pytest.param(k, 2, id="{}x{}x{}-n{}-k{}s{}-{}-tf32".format(*k)) for k in PRODUCTION_TF32])
def test_production_shape_exact(key, rule, workdir):
    """rule 0: the bf16 engine; rule 2: the GPU INT8 rule's tf32 layers, f32 in and out"""
    import torch
    net, i = production_net(key, rule=rule)
    stem = key[-1] == "stem_s2"
    x = net.images(16, 0, 16) if stem else net.images()
    m = util.load(*exact_model.write_net(net, workdir, "prod{}_{}x{}x{}_n{}_k{}s{}_{}".format(rule or "", *key)), net.batch,
                  quantized=net.quantized, fuse=net.fuse)
    p = m.tc_plan(i, quantized=rule)
    assert p.get("kernel") == KERNEL_OF[net.kern[i]] and p["kind"] == ("tf32" if rule else "bf16"), (key, p)
    if net.kern[i] == "reg":
        assert p["BN"] >= min(64, key[3]), (key, p)     # the production tiles: 64 to 256 filters (32 at n = 32)
    if key[-1] == "slice":
        assert p["out_ldc"] == 2 * key[3], (key, p)
    for j, kern in net.kern.items():
        assert m.tc_plan(j, quantized=rule).get("kernel") == KERNEL_OF[kern], (key, j)
    # the expected outputs, each convolution's premise checked, before the network runs
    dev = torch.device("cuda")
    cur = torch.as_tensor(x, device=dev).permute(0, 2, 3, 1).double()
    shapes = net.shapes()
    outs = {}
    for j in sorted(net.params):
        w, b = net.params[j]
        if stem and j == 0:
            cur = cur.to(torch.bfloat16).double()
        res = outs[0] if key[-1] == "shortcut" and j == i else None
        outs[j] = _t_layer(cur, w, b, shapes[j], net.kern[j], res=res, bf16=not rule and key[-1] != "yolo")
        cur = outs[j].double()
    del cur
    m.predict(x, quantized=rule)
    for j, out in outs.items():
        if key[-1] == "yolo":
            got = torch.as_tensor(m.detection_outputs()[j + 1], device=dev)
            v = out.permute(0, 3, 1, 2)
            raw = torch.as_tensor(np.isin(np.arange(v.shape[1]) % 85, (2, 3)), device=dev)
            assert torch.equal(got[:, raw].contiguous().view(torch.int32), v[:, raw].contiguous().view(torch.int32)), key
            vs = v[:, ~raw].double()
            sg = torch.sigmoid(vs)
            assert bool(((got[:, ~raw].double() - sg).abs() / sg <= (4.5 + torch.floor((1.173 * vs).abs())) * 2.0 ** -23).all()), key
        elif key[-1] == "shortcut" and j == i:
            assert _t_bits_equal(m.fetch_layer(j + 1), out), key      # the fused shortcut's output
        elif not (stem and j == 0):                                   # k_stem_s2_tc never writes the stem output
            assert _t_bits_equal(m.fetch_layer(j, quantized=rule), out), (key, j)
    del m
    torch.cuda.empty_cache()
