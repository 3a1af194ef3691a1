"""The C-ABI library loads without a GPU and exports every symbol include/yolo2_light_b200.h declares; compute
entry points fail loudly (no CPU fallback) when no sm_90 device is present."""
import ctypes
import os
import re

import numpy as np
import pytest

import ybtest_util as util

HEADER = os.path.join(util.ROOT, "include", "yolo2_light_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(yb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from yolo2_light_b200 import api
    L = ctypes.CDLL(api.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(L, s), f"{s} declared in the header but not exported"
    for s in api.EXPORTED_SYMBOLS:
        assert s in syms, f"{s} bound in api.py but not declared in the header"


def test_header_cites_reference_for_each_replaced_entry_point():
    text = open(HEADER).read()
    for ref_fn in ("parse_network_cfg", "load_weights_upto_cpu", "yolov2_fuse_conv_batchnorm",
                   "calculate_binary_weights", "quantinization_and_get_multipliers", "network_predict_cpu",
                   "network_predict_quantized", "forward_convolutional_layer_cpu", "forward_convolutional_layer_q",
                   "get_network_boxes"):
        assert re.search(ref_fn + r".*?src/[a-z0-9_]+\.c:\d+", text, flags=re.S), ref_fn


def _cuda_available():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_cuda_available(), reason="checks the no-GPU failure mode")
def test_predict_without_gpu_fails_loudly(workdir):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", workdir)
    net = yb.load_network(cfg, wts, batch=1)
    with pytest.raises(yb.YbError, match="no CUDA device|CUDA"):
        net.predict(util.images("tiny64", 1))


def test_set_option_rejects_unknown_names(workdir):
    """An unknown option name, such as the removed "ksplit", fails loudly; the known options still work."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", workdir)
    net = yb.load_network(cfg, wts, batch=1)
    with pytest.raises(yb.YbError, match="unknown option ksplit"):
        net.set_option("ksplit", 1)
    for name, value in (("fuse", 0), ("keep_counts", 1), ("q_index_offset", 0), ("fuse", 1)):
        net.set_option(name, value)


def test_from_layers_roundtrip(workdir):
    """The drop-in path: descriptors exported from one network rebuild an identical one (yb_network_from_layers)."""
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("xnor64", workdir)
    a = yb.load_network(cfg, wts, batch=2, quantized=1)
    descs = [a.layer_desc(i) for i in range(a.n)]
    b = yb.network_from_layers(descs, 2, a.h, a.w, a.c, 1)
    assert b.n == a.n and b.batch == 2
    for i in range(a.n):
        la, lb = a.layer(i), b.layer(i)
        for k, v in la.items():
            if k in ("scales", "rolling_mean", "rolling_variance"):
                continue   # folded away: not part of a prepared layer
            if isinstance(v, np.ndarray):
                assert np.array_equal(v, lb[k]), (i, k)
            elif k not in ("quantized",):
                assert v == lb[k], (i, k, v, lb[k])
