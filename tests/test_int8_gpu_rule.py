"""The GPU build's INT8 mode (YB_QUANT_GPU, network_predict_gpu_cudnn_quantized) on the host side: the layer rule against the
reference's parser, the saturating input conversion on its edges, the integer part of the oracle against the reference's own
im2col_cpu_int8 + gemm_nn_int8_int32, and the loud failure of every forward entry point without a device."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import rule_oracle as ro
import ybtest_util as util

ASSETS = sorted(glob.glob(os.path.join(util.GOLDEN, "assets", "*.cfg")))


def _our_flags(cfg):
    import yolo2_light_b200 as yb
    net = yb.parse_network_cfg(cfg, 1, 1)
    return {i for i, l in enumerate(net.layers) if l["type_name"] == "CONVOLUTIONAL" and l["quantized"]}


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("cfg", ASSETS, ids=[os.path.basename(p) for p in ASSETS])
def test_layer_rule_matches_reference_parser(cfg):
    """parse_convolutional's l.quantized (additionally.c:3557-3559) with the [yolo] latch (:3996-4003), cfg parsed with
    quantized = 1: our parser flags the same convolutions."""
    from oracle import ref
    rnet = ref.RefNet(cfg, None, 1, 1, 0)
    theirs = {i for i, l in enumerate(rnet.layers) if l["type_name"] == "CONVOLUTIONAL" and l["quantized"]}
    assert _our_flags(cfg) == theirs


def test_layer_rule_of_yolov3_and_yolov3_tiny():
    """yolov3-tiny: the six 3x3/1 backbone layers; yolov3: layer 1 (3x3/2 at index 1), the 23 backbone 3x3/1 layers, 76
    and 78, nothing from layer 80 on."""
    tiny = _our_flags(os.path.join(util.GOLDEN, "assets", "yolov3-tiny.cfg"))
    assert tiny == {2, 4, 6, 8, 10, 12}
    v3 = _our_flags(os.path.join(util.GOLDEN, "assets", "yolov3.cfg"))
    assert len(v3) == 26 and 1 in v3 and {76, 78} <= v3 and max(v3) == 78
    assert all(i <= 74 or i in (76, 78) for i in v3)


def test_layer_rule_needs_a_quantized_parse():
    import yolo2_light_b200 as yb
    net = yb.parse_network_cfg(os.path.join(util.GOLDEN, "assets", "yolov3-tiny.cfg"), 1, 0)
    assert not any(l["quantized"] for l in net.layers)


def test_gpu_input_conversion_edges():
    """cuda_f32_to_int8 + max_abs (gpu.cu:730-739): truncation, saturation at +-2^31 then the +-127 clamp, NaN -> 0;
    v <= -2^31 is defined as -127.  Where |x * m| >= 32768 the CPU rule's int16 wrap gives a different byte."""
    from oracle import port
    m = np.float32(8.0)
    v = np.array([126.9, -126.9, 127, -127, 32767.5, -32767.5, 40000, -40000, 2.0 ** 31, -(2.0 ** 31)], np.float64)
    x = np.concatenate([(v / float(m)).astype(np.float32), np.array([np.inf, -np.inf, np.nan, -0.0], np.float32)])
    got = ro.quantize_input_gpu(x, m)
    exp = np.array([126, -126, 127, -127, 127, -127, 127, -127, 127, -127, 127, -127, 0, 0], np.int8)
    assert np.array_equal(got, exp), got
    cpu = port.quantize_input(x, m)
    assert np.array_equal(cpu[:4], got[:4])
    assert cpu[6] == -127 and cpu[7] == 127 and got[6] == 127 and got[7] == -127   # 40000 wraps through int16 on the CPU


def test_gpu_conv_epilogue_formula():
    """conv_int8_gpu: y = act((float)acc * (1 / (m_in * m_w)) + bias), one rounded multiply, one rounded add.  Where the two
    rules' conversions agree (|x * m| < 32768), its accumulators are those of the CPU rule's oracle (oracle/port.py, pinned
    against the reference)."""
    from oracle import port
    rng = np.random.default_rng(3)
    x = rng.normal(0, 2, (2, 5, 6, 7)).astype(np.float32)
    w = rng.integers(-127, 128, (4, 5, 3, 3), dtype=np.int8)
    b = rng.normal(0, 1, 4).astype(np.float32)
    mi, mw = np.float32(11.0), np.float32(37.0)
    for stride in (1, 2):
        _, a_cpu = port.conv_int8(x, w, b, mi, mw, 4, 3, stride, 1, 3, want_acc=True)
        _, a_gpu = ro.conv_int8_gpu(x, w, b, mi, mw, 4, 3, stride, 1, 3, want_acc=True)
        assert np.array_equal(a_cpu, a_gpu), stride
    for act in (3, 7, 0):
        y, acc = ro.conv_int8_gpu(x, w, b, mi, mw, 4, 3, 1, 1, act, want_acc=True)
        alpha = np.float32(1) / (mi * mw)
        z = (acc.astype(np.float32) * alpha).astype(np.float32) + b[None, :, None, None]
        if act == 7:
            z = np.where(z > 0, z, (0.1 * z.astype(np.float64)).astype(np.float32))
        elif act == 0:
            z = (1.0 / (1.0 + np.exp(-z.astype(np.float64)))).astype(np.float32)
        assert util.bits_equal(y, z), act


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("c,h,w,n,size,stride", [(3, 9, 7, 5, 3, 1), (5, 8, 8, 7, 3, 2), (16, 6, 5, 9, 3, 1),
                                                  (13, 7, 9, 4, 1, 1), (6, 11, 10, 3, 3, 2)])
def test_int8_accumulators_match_reference_gemm(c, h, w, n, size, stride):
    """The reference's own im2col_cpu_int8 (..._quantized.c:186) + gemm_nn_int8_int32 (:493), scalar build, over the
    GPU-converted input and reference-prepared weights_int8, give conv_int8_gpu's accumulators.  gemm_nn_int8_int32
    stores clamp(+-32767, sum / 32); with ALPHA = 32 that is the sum itself while |sum| <= 32767, which the inputs keep."""
    import tempfile
    from oracle import ref
    from yolo2_light_b200 import cfgs
    secs = [cfgs._net(w, h, [8, 8]), cfgs._conv(c, 3), cfgs._conv(n, size, stride)]
    d = tempfile.mkdtemp()
    cfg = cfgs.write_cfg(secs, os.path.join(d, "g.cfg"))
    wts = cfgs.write_weights(secs, os.path.join(d, "g.weights"), seed=c * 100 + n)
    rnet = ref.RefNet(cfg, wts, 1, 1, 7)
    L = rnet.layers[1]
    K = c * size * size
    wq = rnet.array(1, "weights_int8", n * K, np.int8)
    m_in = L["input_quant_multipler"]
    rng = np.random.default_rng(c + h + n)
    x = rng.normal(0, 0.15, (1, c, h, w)).astype(np.float32) * np.float32(16) / np.float32(m_in)
    x.ravel()[0], x.ravel()[-1] = 1e9 / m_in, -40000 / m_in   # where the two rules' conversions part
    pad = L["pad"]
    _, acc = ro.conv_int8_gpu(x, wq.reshape(n, c, size, size), np.zeros(n, np.float32), m_in, L["weights_quant_multipler"],
                                n, size, stride, pad, 3, want_acc=True)
    assert np.abs(acc).max() <= 32767
    xq = ro.quantize_input_gpu(x, m_in)
    oh, ow = (h + 2 * pad - size) // stride + 1, (w + 2 * pad - size) // stride + 1
    col = np.zeros(K * oh * ow, np.int8)
    out = np.zeros(n * oh * ow, np.int32)
    lib = ref._load("scalar")
    vp = C.c_void_p
    lib.im2col_cpu_int8(xq.ctypes.data_as(vp), c, h, w, size, stride, pad, col.ctypes.data_as(vp))
    lib.gemm_nn_int8_int32(n, oh * ow, K, C.c_int8(32), wq.ctypes.data_as(vp), K, col.ctypes.data_as(vp), oh * ow,
                           out.ctypes.data_as(vp), oh * ow)
    assert np.array_equal(out.reshape(acc.shape), acc)


def _cuda_available():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_cuda_available(), reason="checks the no-GPU failure mode")
def test_gpu_rule_entry_points_fail_loudly_without_a_device(workdir):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", workdir)
    net = yb.load_network(cfg, wts, batch=1, quantized=1)
    x = util.images("tiny64", 1)
    frames = [np.zeros((64, 64, 3), np.uint8)]
    calls = [lambda: net.predict(x, quantized=2),
             lambda: yb.network_predict_b200_cudnn_quantized(net, x),
             lambda: net.forward_convolutional_layer(2, np.zeros((1, 8, 32, 32), np.float32), variant=2),
             lambda: net.submit(x, quantized=2),
             lambda: net.predict_frames_u8(frames, quantized=2),
             lambda: net.submit_frames_u8(frames, 0.25, 0.45, quantized=2),
             lambda: net.predict_batch(x, 1, quantized=2),
             lambda: net.fetch_layer(2, quantized=2)]
    for f in calls:
        with pytest.raises(yb.YbError, match="no CUDA device|0 visible"):
            f()
