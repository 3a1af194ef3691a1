"""The input conversion of an integer convolution (k_int_input) reading a channel slice of a route's buffer at an offset that is
not a multiple of 4 floats: the view is not 16-byte aligned, so the kernel must take its scalar loads, standalone and behind a
2x2 max-pool alike.  GPU box only."""
import numpy as np
import pytest

import ybtest_util as util
from yolo2_light_b200 import cfgs

pytestmark = pytest.mark.gpu


def _secs(kind, pooled):
    """conv A (6 filters) -> conv B -> [2x2 max-pool] -> integer conv, and a route over A and B: with fuse on, A and B are
    channel slices of the route's buffer, B at channel 6 (24 bytes in)"""
    q = kind == "int8"
    secs = [cfgs._net(16, 16, [16] * 8 if q else None), cfgs._conv(6, 3), cfgs._conv(8, 3)]
    if pooled:
        secs.append(("maxpool", {"size": "2", "stride": "2"}))
    secs += [cfgs._conv(16, 3, **({} if q else {"xnor": 1, "bin_output": 1})), ("route", {"layers": "0, 1"}),
             cfgs._conv(18, 1, bn=False, act="linear")]
    return secs


@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("kind", ["int8", "xnor"])
def test_int_input_of_an_unaligned_channel_slice(kind, pooled, workdir):
    q = kind == "int8"
    cfg, wts = util.write_net(workdir, f"int_side_{kind}_{int(pooled)}", _secs(kind, pooled), 31)
    B = 2
    x = cfgs.synthetic_images(B, 3, 16, 16, seed=32)
    ic = 3 if pooled else 2          # the integer convolution behind conv B
    res = []
    for fuse in (0, 1):
        net = util.load(cfg, wts, B, quantized=int(q), fuse=fuse, keep_counts=True)
        net.predict(x, quantized=q)
        ops = [(li, k) for li, k, _ in net.profile(quantized=q)]
        ints = [i for i, l in enumerate(net.layers)
                if l["type_name"] == "CONVOLUTIONAL" and (l["xnor"] or (q and i >= 1 and l["activation"] != 3))]
        assert ic in ints, ints
        res.append((ops, [net.fetch_counts(i, quantized=q) for i in ints], net.fetch_layer(ic, quantized=q)))
    ops0, ops1 = res[0][0], res[1][0]
    conv = "quantize" if q else "binarize"
    if pooled:
        # fuse = 1: the max-pool writes the integer layer's input itself (k_int_input behind the 2x2 window)
        assert (2, "maxpool") in ops1 and (ic, conv) not in ops1 and (ic, conv) in ops0, (ops0, ops1)
    else:
        assert (ic, conv) in ops0 and (ic, conv) in ops1, (ops0, ops1)
    for a, b in zip(res[0][1], res[1][1]):
        assert np.array_equal(a, b)
    assert np.array_equal(res[0][2].view(np.uint32), res[1][2].view(np.uint32))
