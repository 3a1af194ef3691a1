"""CPU restatement of the reference's GPU INT8 mode (network_predict_gpu_cudnn_quantized, yolov2_forward_network_gpu.cu:576),
for the tests of YB_QUANT_GPU: the input conversion, the INT8 convolution and a whole-network runner that follows
forward_network_gpu_cudnn_quantized's loop (:494-507) with the oracle's CPU functions (oracle/port.py) for every other layer.

Everything is numpy in IEEE float32 / exact integers, so each value is defined bit for bit:
  conversion  v = x * m rounded once in float32; CUDA's float -> int (truncation, saturating at +-2^31, NaN -> 0); clamp to
              +-127 (cuda_f32_to_int8 + max_abs, gpu.cu:730-739).  v <= -2^31 gives -127: max_abs read without overflow; what
              the reference binary does with abs(INT_MIN) depends on its compiler.
  convolution acc = sum wq * xq over the in-image taps, exact (float64 products and sums of s8 values stay below 2^53);
              y = (float)acc * ALPHA1, ALPHA1 = 1 / (m_in * m_w) (:200); y += bias; then activate() of the scalar build
              (additionally.h:85-91) -- one rounded multiply and one rounded add.
"""
from typing import List, Optional, Sequence

import numpy as np

from oracle import port

F32 = np.float32


def quantize_input_gpu(x, mult) -> np.ndarray:
    v = (np.asarray(x, F32) * F32(mult)).astype(np.float64)   # the float32 product, exactly
    v = np.trunc(np.nan_to_num(v, nan=0.0))                     # truncation; NaN -> 0 (+-inf saturate below)
    return np.clip(v, -127, 127).astype(np.int8)


def activate(y: np.ndarray, act: int) -> np.ndarray:
    y = np.asarray(y, F32)
    if act == port.LEAKY:
        return np.where(y > 0, y, (0.1 * y.astype(np.float64)).astype(F32))
    if act == 0:   # LOGISTIC
        return (1.0 / (1.0 + np.exp(-y.astype(np.float64)))).astype(F32)
    if act == 1:   # RELU
        return y * (y > 0)
    return y


def conv_int8_gpu(x, weights_int8, biases, input_mult, weights_mult, n, size, stride, pad, activation, want_acc=False):
    x = np.asarray(x, F32)
    b, c, h, w = x.shape
    oh, ow = (h + 2 * pad - size) // stride + 1, (w + 2 * pad - size) // stride + 1
    wq = np.asarray(weights_int8, np.int8).reshape(n, c * size * size).astype(np.float64)
    acc = np.empty((b, n, oh, ow), np.int32)
    for k in range(b):
        xq = np.pad(quantize_input_gpu(x[k], input_mult).astype(np.float64), ((0, 0), (pad, pad), (pad, pad)))
        cols = np.empty((c, size, size, oh, ow), np.float64)   # K ordered (c, ky, kx), the weights' order
        for ky in range(size):
            for kx in range(size):
                cols[:, ky, kx] = xq[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride]
        acc[k] = (wq @ cols.reshape(c * size * size, oh * ow)).astype(np.int64).reshape(n, oh, ow)
    alpha1 = F32(1) / (F32(input_mult) * F32(weights_mult))
    y = acc.astype(F32) * alpha1
    y = y + np.asarray(biases, F32).reshape(1, n, 1, 1)
    out = activate(y, activation)
    return (out, acc) if want_acc else out


def run_network_gpu(layers: Sequence[dict], x: np.ndarray) -> List[Optional[np.ndarray]]:
    """forward_network_gpu_cudnn_quantized: convolution i is INT8 (conv_int8_gpu) iff its `quantized` flag is set; every other
    layer is the oracle's CPU function, as port.run_network computes it without an INT8 rule.  Returns every layer's output."""
    outs: List[Optional[np.ndarray]] = []
    cur = np.ascontiguousarray(x, F32)
    for l in layers:
        t = l["type"]
        if t == port.CONVOLUTIONAL:
            if l["quantized"]:
                o = conv_int8_gpu(cur, l["weights_int8"], l["biases"], l["input_quant_multipler"], l["weights_quant_multipler"],
                                  l["n"], l["size"], l["stride"], l["pad"], l["activation"])
            elif l["xnor"]:
                o = port.conv_xnor(cur, l["weights"], l["biases"], l["mean_arr"], l["n"], l["size"], l["activation"])
            else:
                o = port.conv_fp32(cur, l["weights"], l["biases"], l["n"], l["size"], l["stride"], l["pad"], l["activation"])
        elif t == port.MAXPOOL:
            o = port.maxpool(cur, l["size"], l["stride"], l["pad"])
        elif t == port.ROUTE:
            o = np.concatenate([outs[int(j)] for j in l["input_layers"]], axis=1)
        elif t == port.UPSAMPLE:
            o = port.upsample(cur, l["stride"], l["scale"])
        elif t == port.SHORTCUT:
            o = port.shortcut(cur, outs[l["index"]], l["activation"])
        elif t == port.REORG:
            o = port.reorg(cur, l["stride"])
        elif t == port.YOLO:
            o = port.yolo(cur, l["n"], l["classes"])
        elif t == port.REGION:
            o = port.region(cur, l["n"], l["classes"], l["coords"], l["softmax"])
        else:
            o = cur
        outs.append(o)
        cur = o
    return outs
