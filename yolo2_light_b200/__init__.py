"""yolo2_light_b200 -- Hopper (sm_90a, H100) forward-inference engine behind the C surface of AlexeyAB/yolo2_light.

The product is ``libyolo2_light_b200.so`` (C ABI in ``include/yolo2_light_b200.h``); this package is its ctypes
mirror plus generators for the model definitions / synthetic weights used by the tests and the benchmark.
"""
from . import cfgs  # noqa: F401
from .api import (  # noqa: F401
    YB_PREC_BF16_TC, YB_PREC_FP32, YB_QUANT_CPU, YB_QUANT_GPU, YB_QUANT_NONE, YB_XNOR_CPU, YB_XNOR_GPU, LayerDesc, Network, PinnedBuffer, YbError,
    calculate_binary_weights, lib, load_network, load_weights_upto_cpu, network_from_layers,
    network_predict_b200, network_predict_b200_cudnn_quantized, network_predict_b200_quantized, parse_network_cfg,
    quantinization_and_get_multipliers, yolov2_fuse_conv_batchnorm,
)
