"""Pins the CPU restatement (oracle/yolo_oracle.c) against the UNMODIFIED reference (oracle/_ref/
libyolo2ref_scalar.so, built from the reference sources by oracle/Makefile): whole networks, every layer, bit-for-bit."""
import numpy as np
import pytest

import ybtest_util as util

pytestmark = pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libyolo2ref_scalar.so not built")


def _ref_and_port(name, workdir, quantized, batch=1):
    import yolo2_light_b200 as yb
    from oracle import port, ref
    cfg, wts = util.model_files(name, workdir)
    x = util.images(name, batch)
    rnet = ref.RefNet(cfg, wts, batch, quantized, 7)
    rnet.predict(x)
    net = yb.load_network(cfg, wts, batch=batch, quantized=quantized)
    outs = port.run_network(net.layers, x, quantized=bool(quantized))
    return rnet, outs


@pytest.mark.parametrize("name,quantized", [("tiny64", 0), ("tiny64", 1), ("xnor64", 0), ("v3_32", 0),
                                            ("spp32", 0), ("v2voc32", 0), ("tinyvoc64", 1), ("v3_32", 1),
                                            ("tiny_w96_h64", 0), ("tiny_w96_h64", 1), ("v3_w64_h96", 0),
                                            ("edges_yolo_w40_h24", 0), ("edges_region_w26_h22", 0)])
def test_whole_network_bit_exact(name, quantized, workdir):
    """Same cfg, same generated .weights, same image -> every layer output of the restatement equals the
    reference's l.output bit-for-bit (FP32 conv: identical k-ascending float accumulation; XNOR / INT8: exact
    integers + identical float epilogue; small layers: copies / compares / libm)."""
    rnet, outs = _ref_and_port(name, workdir, quantized)
    for i, o in enumerate(outs):
        r = rnet.output(i)
        assert o.size == r.size, (i, o.shape, r.shape)
        assert util.bits_equal(o.reshape(r.shape), r), (
            f"{name} q={quantized} layer {i} {rnet.layers[i]['type_name']}: "
            f"max abs diff {np.abs(o.reshape(r.shape) - r).max()}")


def test_batch_two_fp32(workdir):
    """The reference's FP32/XNOR loops handle l.batch > 1 (yolov2_forward_network.c:111, :212); so does the port."""
    rnet, outs = _ref_and_port("xnor64", workdir, 0, batch=2)
    for i, o in enumerate(outs):
        r = rnet.output(i)
        assert util.bits_equal(o.reshape(r.shape), r), i


@pytest.mark.parametrize("name", ["edges_yolo_w40_h24", "edges_region_w26_h22"])
def test_batch_three_edge_shapes(name, workdir):
    """The edge geometries at batch 3, where the reference's reorg of a size its stride does not divide reads each image
    from a flat offset inside the images before it (yolov2_forward_network.c:359-366)"""
    rnet, outs = _ref_and_port(name, workdir, 0, batch=3)
    for i, o in enumerate(outs):
        r = rnet.output(i)
        assert util.bits_equal(o.reshape(r.shape), r), (name, i, rnet.layers[i]["type_name"])


def test_quantize_input_matches_reference_cast():
    """(int16_t)(x*mult) with x86 semantics, clamp +-127 (yolov2_forward_network_quantized.c:556-560), including
    values around the truncation boundaries and large magnitudes."""
    from oracle import port
    x = np.array([0.0, 0.49, -0.49, 1.0, -1.0, 7.999, -7.999, 126.9, 127.2, -127.2, 300.0, -300.0,
                  32767.9, 32768.5, -32769.5, 65536.0 + 5, 1e9, -1e9, 1e20, np.nan], np.float32)
    q = port.quantize_input(x, 1.0)
    exp = []
    for v in x:
        f = np.float32(v)
        if not (f > -2147483648.0 and f < 2147483648.0):
            i = -2147483648
        else:
            i = int(f)
        s = ((i & 0xffff) ^ 0x8000) - 0x8000
        exp.append(max(-127, min(127, s)))
    assert q.tolist() == exp


@pytest.mark.parametrize("shape", [(480, 640, 608, 608), (37, 53, 64, 96), (64, 64, 64, 64), (1, 7, 32, 32), (100, 1, 32, 32)])
def test_image_pipeline_port_equals_reference(shape):
    """u8 -> float/255 -> resize_image: the port against the reference's own functions, bit-for-bit."""
    from oracle import port, ref
    h, w, oh, ow = shape
    img = np.random.default_rng(h * 1000 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    assert util.bits_equal(port.load_resize_u8(img, ow, oh), ref.load_resize_u8(img, ow, oh))
