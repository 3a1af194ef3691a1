"""The layers between the convolutions -- max-pool, upsample, route copies, the unfused shortcut, reorg and the unfused
[yolo] / [region] heads -- against the oracle, element by element, in both engine precisions.

Every case runs at batch 3 on a non-square input, once in YB_PREC_FP32 and once in YB_PREC_BF16_TC.  Each layer under test
is checked against the oracle (oracle/port.py) run on the engine's own input, fetched with fetch_layer, so an error is
found in the layer that makes it and not only where it reaches a detection tensor.  A bf16 engine's activations are
bf16 values, so the copies and compares (max-pool, route, reorg, upsample at scale 1) are exact in both precisions, and
the ops that compute (upsample at scale != 1, shortcut) are the oracle's f32 result rounded to bf16.  Each case also
asserts, through Network.op_kernels, which kernel ran the layer: the channel counts and channel offsets of the cases put
the scalar and the 16-byte kernels of max-pool and upsample to work in each precision.

The helpers and the case table run on the CPU; the tests that need a GPU are marked."""
import numpy as np
import pytest

import ybtest_util as util
from ybtest_util import bf16_round, kernel_is, logistic_bound, ulp_diff
from yolo2_light_b200 import cfgs

BATCH = 3
DTYPES = ("f32", "bf16")
ESIZE = {"f32": 4, "bf16": 2}


# ---- the case table -----------------------------------------------------------------------------------------------------
def conv(n, size=3, stride=1, act="leaky"):
    return cfgs._conv(n, size, stride, act=act)


def maxpool(size, stride, padding=None):
    o = {"size": str(size), "stride": str(stride)}
    if padding is not None:
        o["padding"] = str(padding)
    return ("maxpool", o)


def upsample(stride, scale=None):
    o = {"stride": str(stride)}
    if scale is not None:
        o["scale"] = str(scale)
    return ("upsample", o)


def route(*layers):
    return ("route", {"layers": ", ".join(str(j) for j in layers)})


def shortcut(frm, act="linear"):
    return ("shortcut", {"from": str(frm), "activation": act})


def vec16(C, aligned=True):
    """the 16-byte kernel's rule (emit_small): whole 16-byte channel rows at a 16-byte aligned base; every buffer's pixel
    stride is a multiple of 8 channels"""
    return {dt: aligned and C * ESIZE[dt] % 16 == 0 for dt in DTYPES}


class Case:
    """A network (cfg sections after [net]), its fusion option, and the layers under test: layer -> {dtype: kernel}"""

    def __init__(self, h, w, secs, fuse=1):
        self.h, self.w, self.secs, self.fuse = h, w, secs, fuse
        self.kernels = {}

    def expect(self, layer, kernel):
        self.kernels[layer] = kernel if isinstance(kernel, dict) else {dt: kernel for dt in DTYPES}
        return self

    def sections(self):
        return [cfgs._net(self.w, self.h)] + self.secs


def c_maxpool(h, w, C, size, stride, padding=None):
    v = vec16(C)
    return Case(h, w, [conv(C), maxpool(size, stride, padding)]).expect(
        1, {dt: "k_maxpool_vec" if v[dt] else "k_maxpool" for dt in DTYPES})


def c_spp():
    """the SPP block of yolov3-spp: 5, 9 and 13 / 1 max-pools of one layer, concatenated with it"""
    secs = [conv(8), maxpool(5, 1), route(-2), maxpool(9, 1), route(-4), maxpool(13, 1), route(-1, -3, -5, -6)]
    c = Case(7, 11, secs)
    for i in (1, 3, 5):     # each writes its slice of route 6's buffer, at 16-byte aligned channel offsets
        c.expect(i, "k_maxpool_vec")
    return c


def c_maxpool_slice():
    """layer 1 writes channels 6..13 of route 3's buffer: the max-pool's input starts 12 (bf16) or 24 (f32) bytes into a
    pixel, so the scalar kernel runs although C = 8 fills 16-byte rows"""
    secs = [conv(6), conv(8), maxpool(2, 2), route(0, 1)]
    return Case(9, 13, secs, fuse=1).expect(2, "k_maxpool")


def c_upsample(h, w, C, stride, scale):
    v = vec16(C)
    return Case(h, w, [conv(C), upsample(stride, scale)]).expect(
        1, {dt: "k_upsample_vec16" if v[dt] and scale in (None, 1) else "k_upsample" for dt in DTYPES})


def c_upsample_slice():
    secs = [conv(6), conv(8), upsample(2), route(0, 1)]
    return Case(5, 7, secs, fuse=1).expect(2, "k_upsample")


def c_route(fuse):
    """2, 3 and 4 sources of odd channel counts, a source listed twice, a route as a source"""
    secs = [conv(5), conv(7), conv(3), route(0, 1), route(0, 1, 2), route(2, 0, 2, 1), route(3, 2)]
    c = Case(6, 10, secs, fuse=fuse)
    for r in (3, 4, 5, 6):
        c.expect(r, "k_copy_channels")
    return c


# layers copied by each route: every source with fuse=0; with fuse=1 the sources that write their slice themselves
# are not (the first route to list a non-route layer owns it)
ROUTE_COPIES = {0: {3: 2, 4: 3, 5: 4, 6: 2}, 1: {3: 0, 4: 2, 5: 4, 6: 2}}


def c_shortcut_same(act):
    return Case(6, 10, [conv(12), conv(12), shortcut(-2, act)], fuse=0).expect(2, "k_shortcut")


def c_shortcut(kind):
    if kind == "from_2x":        # a stride-2 convolution in front: never fused
        secs = [conv(8), conv(8, 3, 2), shortcut(0, "leaky")]
    elif kind == "from_4x":
        secs = [conv(8), conv(8, 3, 2), conv(8, 3, 2), shortcut(0, "linear")]
    elif kind == "from_half":    # `from` is half the size: the sample branch
        secs = [conv(8, 3, 2), upsample(2), shortcut(0, "leaky")]
    elif kind == "fewer_channels":
        secs = [conv(6), conv(10, 3, 2), shortcut(0, "linear")]
    elif kind == "more_channels":
        secs = [conv(10), conv(6), shortcut(0, "leaky")]
    elif kind == "from_slice":   # `from` is channels 8..15 of route 4's buffer
        secs = [conv(8), conv(8), maxpool(3, 1), shortcut(1, "linear"), route(0, 1)]
    else:
        raise KeyError(kind)
    fuse = 0 if kind == "more_channels" else 1
    return Case(12, 20, secs, fuse=fuse).expect(len(secs) - 1 if kind != "from_slice" else 3, "k_shortcut")


def c_reorg(h, w, stride):
    return Case(h, w, [conv(6), ("reorg", {"stride": str(stride)})]).expect(1, "k_reorg")


def c_yolo(h, w, classes):
    secs = [conv(8), cfgs._conv(3 * (5 + classes), 1, bn=False, act="linear"),
            cfgs._yolo("0,1,2", cfgs.TINY_ANCHORS, 6, classes)]
    return Case(h, w, secs, fuse=0).expect(2, "k_yolo")


def c_region(classes, num, softmax):
    anchors = "1.08,1.19,  3.42,4.41,  6.63,11.38,  9.42,5.11,  16.62,10.52"
    head = ("region", {"anchors": anchors, "classes": str(classes), "coords": "4", "num": str(num), "softmax": str(softmax)})
    secs = [conv(8), cfgs._conv(num * (5 + classes), 1, bn=False, act="linear"), head]
    return Case(6, 8, secs).expect(2, "k_region")


CASES = {
    "maxpool_2s2_7x13_c16": lambda: c_maxpool(7, 13, 16, 2, 2),
    "maxpool_2s1_13x13_c12": lambda: c_maxpool(13, 13, 12, 2, 1),
    "maxpool_spp_7x11": c_spp,
    "maxpool_3s2_pad2_9x10_c6": lambda: c_maxpool(9, 10, 6, 3, 2, 2),
    "maxpool_2s2_pad0_7x13_c12": lambda: c_maxpool(7, 13, 12, 2, 2, 0),
    "maxpool_misaligned_slice": c_maxpool_slice,
    "upsample_s2_c16": lambda: c_upsample(5, 7, 16, 2, None),
    "upsample_s3_c12": lambda: c_upsample(5, 7, 12, 3, 1),
    "upsample_s2_scale0.5_c16": lambda: c_upsample(5, 7, 16, 2, 0.5),
    "upsample_s3_scale0.5_c6": lambda: c_upsample(4, 7, 6, 3, 0.5),
    "upsample_slice": c_upsample_slice,
    "route_fuse0": lambda: c_route(0),
    "route_fuse1": lambda: c_route(1),
    **{f"shortcut_same_{a}": (lambda a=a: c_shortcut_same(a)) for a in ("linear", "leaky", "relu", "logistic")},
    **{f"shortcut_{k}": (lambda k=k: c_shortcut(k)) for k in ("from_2x", "from_4x", "from_half", "fewer_channels",
                                                              "more_channels", "from_slice")},
    "reorg_s2_13x13": lambda: c_reorg(13, 13, 2),
    "reorg_s2_6x10": lambda: c_reorg(6, 10, 2),
    "reorg_s3_9x7": lambda: c_reorg(9, 7, 3),
    "yolo_c1_7x9": lambda: c_yolo(7, 9, 1),
    "yolo_c80_5x7": lambda: c_yolo(5, 7, 80),
    "region_softmax1": lambda: c_region(20, 5, 1),
    "region_softmax0": lambda: c_region(3, 2, 0),
}


# ---- comparisons --------------------------------------------------------------------------------------------------------
def expf_bounds(softmax_n):
    """Bounds, relative to the exact value, on k_region's logistic 1 / (1 + expf(-v)) and on its softmax over softmax_n
    classes, from the CUDA C Programming Guide's maximum error of expf (2 ulp, full range) and IEEE rounding of +, / (u =
    2^-24 each).  Logistic: expf within 2 ulp <= 4u relative, and 1 + e has at most that relative error plus its own
    rounding, then the division rounds once: 4u + u + u.  Softmax over exp(d_k) with the f32 differences d_k = v_k - max:
    each e_k within 4u, their sum within 4u + (n - 1) u from the n - 1 rounded additions (first order), the quotient within
    4u + 4u + (n - 1) u + u.  One more u absorbs the second-order terms."""
    u = 2.0 ** -24
    return (7 * u), (4 + 4 + (softmax_n - 1) + 1 + 1) * u


def check_layer(m, i, L, layers, bf16, q=False):
    """layer i of the engine against the oracle on the engine's input; returns what was compared"""
    from oracle import port
    t = L["type_name"]
    got = m.fetch_layer(i, quantized=q)
    fetch = lambda j: m.fetch_layer(j, quantized=q)
    rnd = bf16_round if bf16 else (lambda a: a)
    if t in ("MAXPOOL", "REORG"):
        assert util.bits_equal(got, util.oracle_layer(L, i, fetch(i - 1), int(q))[0]), i
    elif t == "UPSAMPLE":
        assert util.bits_equal(got, rnd(util.oracle_layer(L, i, fetch(i - 1), int(q))[0])), i
    elif t == "ROUTE":
        assert util.bits_equal(got, np.concatenate([fetch(int(j)) for j in L["input_layers"]], axis=1)), i
    elif t == "SHORTCUT":
        exp = rnd(util.oracle_layer(L, i, fetch(i - 1), int(q), frm=fetch(L["index"]))[0])
        d = ulp_diff(got, exp, bf16)
        assert d.max() <= (1 if L["activation"] == 0 else 0), (i, int(d.max()), int((d > 0).sum()))
    elif t == "YOLO":
        head = fetch(i - 1)
        per = 4 + L["classes"] + 1
        raw = np.isin(np.arange(head.shape[1]) % per, (2, 3))
        assert util.bits_equal(got[:, raw], head[:, raw]), i
        if bf16:     # the __expf logistic of the bf16 networks
            v = head[:, ~raw]
            sg = 1.0 / (1.0 + np.exp(-v.astype(np.float64)))
            err = np.abs(got[:, ~raw] - sg) / sg
            assert np.all(err <= logistic_bound(v)), (i, float(err.max()))
        else:        # the double-precision logistic of the reference
            d = ulp_diff(got[:, ~raw], port.yolo(head, L["n"], L["classes"])[:, ~raw], False)
            assert d.max() <= 1, (i, int(d.max()))
    elif t == "REGION":
        head = fetch(i - 1)
        n, classes, size = L["n"], L["classes"], 4 + L["classes"] + 1
        assert L["coords"] == 4
        B = head.shape[0]
        v = head.reshape(B, n * size, -1).transpose(0, 2, 1).reshape(B, -1, size).astype(np.float64)   # [b][cell, anchor][entry]
        g = got.reshape(B, -1, size)
        assert util.bits_equal(g[..., :4], v[..., :4].astype(np.float32)), i
        lb, sb = expf_bounds(classes)
        sg = 1.0 / (1.0 + np.exp(-v[..., 4]))
        assert np.all(np.abs(g[..., 4] - sg) <= lb * sg), (i, float((np.abs(g[..., 4] - sg) / sg).max()))
        cls = v[..., 5:].astype(np.float32)
        if L["softmax"]:
            dk = (cls - cls.max(axis=-1, keepdims=True)).astype(np.float64)   # the f32 differences both sides compute
            e = np.exp(dk)
            sm = e / e.sum(axis=-1, keepdims=True)
            err = np.abs(g[..., 5:] - sm)
            assert np.all(err <= sb * sm), (i, float((err / sm).max()))
        else:
            assert util.bits_equal(g[..., 5:], cls), i
    else:
        raise AssertionError(f"layer {i}: no check for {t}")
    return t


# ---- CPU tests ----------------------------------------------------------------------------------------------------------
def test_cases_run_both_kernels_of_maxpool_and_upsample():
    """in each precision, the table runs the scalar and the 16-byte kernel of max-pool and of upsample"""
    for dt in DTYPES:
        ran = {CASES[name]().kernels[i][dt] for name in CASES for i in CASES[name]().kernels}
        for k in ("k_maxpool", "k_maxpool_vec", "k_upsample", "k_upsample_vec16"):
            assert k in ran, (dt, k)


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_shapes(name):
    """non-square inputs, and every layer under test of a kind check_layer knows"""
    c = CASES[name]()
    shapes = cfgs.conv_shapes(c.sections())
    assert c.h != c.w or name == "reorg_s2_13x13" or name == "maxpool_2s1_13x13_c12"
    for i in c.kernels:
        assert shapes[i]["type"] in ("maxpool", "upsample", "route", "shortcut", "reorg", "yolo", "region"), (name, i)


def test_ulp_diff():
    a = np.array([1.0, -1.0, 0.0, -0.0, 2.0], np.float32)
    b = np.nextafter(a, np.float32(np.inf))
    assert ulp_diff(a, b, False).tolist() == [1] * 5
    assert ulp_diff(np.float32(0.0), np.float32(-0.0), False) == 0
    assert ulp_diff(bf16_round(np.float32(1.0)), np.float32(1.0078125), True) == 1


# ---- GPU tests ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_small_layer(name, dt, workdir):
    import yolo2_light_b200 as yb
    case = CASES[name]()
    m = util.load(*util.write_net(workdir, f"small_{name}", case.sections(), sum(map(ord, name))), BATCH,
                  precision=yb.YB_PREC_FP32 if dt == "f32" else yb.YB_PREC_BF16_TC, fuse=case.fuse)
    ops = [op for op in m.op_kernels() if op[2] is None or "k_nhwc_to_nchw_f32" not in op[2]]   # not the last layer's NCHW copy
    for i, kern in case.kernels.items():
        mine = [k for (j, _, k) in ops if j == i]
        if name.startswith("route") and ROUTE_COPIES[case.fuse][i] == 0:
            assert not mine, (name, dt, i, mine)     # every source writes its own slice
            continue
        assert mine and all(kernel_is(k, kern[dt]) for k in mine), (name, dt, i, mine)
        # the templated kernels: instantiated for the layer's activation dtype
        assert all(("__nv_bfloat16" in k) == (dt == "bf16" and kern[dt] not in ("k_yolo", "k_region")) for k in mine), \
            (name, dt, i, mine)
    if name.startswith("route"):
        for r, n in ROUTE_COPIES[case.fuse].items():
            assert sum(1 for (j, kind, _) in ops if j == r and kind == "route_copy") == n, (name, dt, r, ops)
    m.predict(cfgs.synthetic_images(BATCH, 3, case.h, case.w, seed=len(name)))
    layers = m.layers
    for i in case.kernels:
        check_layer(m, i, layers[i], layers, dt == "bf16")


@pytest.mark.gpu
def test_shortcut_whose_scales_differ_in_width_and_height_is_rejected(workdir):
    """56 x 50 input: layer 0 is 56 x 50, three 3x3/2 convolutions make 28 x 25, 14 x 13 and 7 x 7, an upsample 14 x 14.  A
    shortcut from layer 0 onto it would take stride 56 / 14 = 4 from the widths and read rows 0, 4, .., 52 of a 50-row
    tensor; the reference asserts stride == h1 / h2 = 3 and stops.  The engine refuses the network in its layer plan."""
    import yolo2_light_b200 as yb
    secs = [cfgs._net(56, 50), conv(8), conv(8, 3, 2), conv(8, 3, 2), conv(8, 3, 2), upsample(2), shortcut(0)]
    m = util.load(*util.write_net(workdir, "shortcut_aspect", secs, 1), 2)
    assert (m.layer(5)["out_w"], m.layer(5)["out_h"]) == (14, 14)
    for prec in (yb.YB_PREC_BF16_TC, yb.YB_PREC_FP32):
        m.set_precision(prec)
        with pytest.raises(yb.YbError, match="shortcut from layer 0 .56x50. onto 14x14"):
            m.op_kernels()


@pytest.mark.gpu
def test_region_with_coords_other_than_4_is_rejected(workdir):
    """The reference's forward takes the objectness at entry 4 and the classes from entry 5 whatever coords is, and so do
    both decoders: a [region] layer with coords != 4 is refused"""
    import yolo2_light_b200 as yb
    head = ("region", {"anchors": "1,1, 2,2", "classes": "3", "coords": "5", "num": "2", "softmax": "1"})
    secs = [cfgs._net(8, 6), conv(8), cfgs._conv(2 * (5 + 1 + 3), 1, bn=False, act="linear"), head]
    m = util.load(*util.write_net(workdir, "region_coords5", secs, 2), 1)
    with pytest.raises(yb.YbError, match=r"\[region\] coords=5 is not supported"):
        m.op_kernels()
