"""CPU restatement of the reference GPU build's XNOR arithmetic (forward_convolutional_layer_gpu_cudnn,
yolov2_forward_network_gpu.cu:23-139), for the tests of YB_XNOR_GPU: the per-layer path choice, both paths and a
whole-network runner.

Everything is numpy in IEEE float32 / exact integers, so each value is defined bit for bit:
  path A  c % 32 == 0, any geometry: input bit x > 0, out-of-image taps -1, dot = 2*count - K (exact);
          y = fmaf((float)dot, mean, bias), correctly rounded once (fmaf_f32 below); leaky `y >= 0 ? y : 0.1f*y` in float,
          any other activation after it.  A same-shape [shortcut] behind it is `from + v`, v the leaky-only value, with no
          activation.
  path B  c < 32: s = sum sign(w) * (x >= 0 ? +1 : -1), out-of-image taps 0 (exact); y = act((float)s * mean + bias)
          with a rounded multiply and a rounded add.
  act     leaky in float (0.1f * y), logistic in double as every other layer of the engine, relu and linear exact.
"""
from fractions import Fraction
from typing import List, Optional, Sequence

import numpy as np

import gpu_rule_oracle as gro
from oracle import port

F32 = np.float32


class Rejected(ValueError):
    """A network the GPU XNOR rule does not run."""


def fmaf_f32(a, b, c) -> np.ndarray:
    """fmaf(a, b, c) of float32 arrays, correctly rounded.  a * b is exact in float64 (two 24-bit significands); the sum
    s = fl64(a*b + c) with its exact error e (TwoSum) is the exact result s + e.  Rounding s to float32 gives the right
    answer unless s lies exactly on a float32 midpoint, where the sign of e decides (e == 0: ties to even, as s rounds)."""
    a = np.asarray(a, F32).astype(np.float64)
    b = np.asarray(b, F32).astype(np.float64)
    c = np.asarray(c, F32).astype(np.float64)
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(F32)
    r64 = r.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        toward = np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(F32)
        other = np.nextafter(r, toward)
        mid = (r64 + other.astype(np.float64)) / 2
        tie = (s != r64) & (s == mid) & (e != 0)
        up = (e > 0) == (other.astype(np.float64) > r64)   # e pushes the exact value toward `other`
    return np.where(tie & up, other, r).astype(F32)


def fmaf_exact(a, b, c) -> np.float32:
    """One fmaf by exact rational arithmetic, rounded to float32 to nearest-even (finite, normal results)."""
    v = Fraction(float(F32(a))) * Fraction(float(F32(b))) + Fraction(float(F32(c)))
    if v == 0:
        return F32(0.0)
    lo = F32(float(v))                       # within one float32 step of v
    cands = sorted({np.nextafter(lo, F32(-np.inf)), lo, np.nextafter(lo, F32(np.inf))}, key=float)
    best = min(cands, key=lambda t: (abs(Fraction(float(t)) - v), int(np.array(t, F32).view(np.uint32)) & 1))
    return F32(best)


def act_gpu(y, act: int) -> np.ndarray:
    y = np.asarray(y, F32)
    if act == port.LEAKY:
        return np.where(y >= 0, y, F32(0.1) * y).astype(F32)
    return gro.activate(y, act)


def _cols(xp, size, stride, oh, ow):
    c = xp.shape[0]
    cols = np.empty((c, size, size, oh, ow), np.float64)   # K ordered (c, ky, kx), the weights' order
    for ky in range(size):
        for kx in range(size):
            cols[:, ky, kx] = xp[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride]
    return cols.reshape(c * size * size, oh * ow)


def _signed_sum(b_in, weights, n, size, stride, pad, pad_value):
    """sum sign(w) * b over the taps, exact: b_in is +-1 per element, out-of-image taps pad_value"""
    b, c, h, w = b_in.shape
    oh, ow = (h + 2 * pad - size) // stride + 1, (w + 2 * pad - size) // stride + 1
    ws = np.where(np.asarray(weights, F32).reshape(n, c * size * size) > 0, 1.0, -1.0)
    out = np.empty((b, n, oh, ow), np.int32)
    for k in range(b):
        xp = np.pad(b_in[k], ((0, 0), (pad, pad), (pad, pad)), constant_values=pad_value)
        out[k] = (ws @ _cols(xp, size, stride, oh, ow)).astype(np.int64).reshape(n, oh, ow)
    return out


def bin_dot(x, weights, n, size, stride, pad) -> np.ndarray:
    """Path A's dot = 2*count - K: input bit x > 0, out-of-image taps -1."""
    return _signed_sum(np.where(np.asarray(x, F32) > 0, 1.0, -1.0), weights, n, size, stride, pad, -1.0)


def pm1z_sum(x, weights, n, size, stride, pad) -> np.ndarray:
    """Path B's s: b(x) = x >= 0 ? +1 : -1 (NaN: -1), out-of-image taps 0."""
    return _signed_sum(np.where(np.asarray(x, F32) >= 0, 1.0, -1.0), weights, n, size, stride, pad, 0.0)


def conv_xnor_a(x, L, want_raw=False, leaky_only=False):
    n = L["n"]
    dot = bin_dot(x, L["weights"], n, L["size"], L["stride"], L["pad"])
    mean = np.asarray(L["mean_arr"], F32).reshape(1, n, 1, 1)
    bias = np.asarray(L["biases"], F32).reshape(1, n, 1, 1)
    v = fmaf_f32(dot.astype(F32), np.broadcast_to(mean, dot.shape), np.broadcast_to(bias, dot.shape))
    act = L["activation"]
    y = act_gpu(v, act) if (act == port.LEAKY or not leaky_only) else v
    return (y, dot) if want_raw else y


def conv_xnor_b(x, L, want_raw=False):
    n = L["n"]
    s = pm1z_sum(x, L["weights"], n, L["size"], L["stride"], L["pad"])
    mean = np.asarray(L["mean_arr"], F32).reshape(1, n, 1, 1)
    bias = np.asarray(L["biases"], F32).reshape(1, n, 1, 1)
    y = act_gpu((s.astype(F32) * mean).astype(F32) + bias, L["activation"])
    return (y, s) if want_raw else y


def _same_shape_shortcut(S) -> bool:
    return S["type_name"] == "SHORTCUT" and S["w"] == S["out_w"] and S["h"] == S["out_h"] and S["c"] == S["out_c"]


def xnor_paths(layers: Sequence[dict], int8_gpu: bool = False) -> dict:
    """layer -> "A" or "B" for every XNOR convolution the rule runs as XNOR (int8_gpu: the l.quantized ones run INT8);
    raises Rejected where the engine refuses the network."""
    paths = {}
    for i, L in enumerate(layers):
        if L["type_name"] != "CONVOLUTIONAL" or not L["xnor"]:
            continue
        nxt = layers[i + 1] if i + 1 < len(layers) else None
        sc = nxt is not None and _same_shape_shortcut(nxt)
        c = L["c"]
        if c >= 32 and c % 32:
            raise Rejected(f"layer {i}: c = {c}")
        int8 = int8_gpu and L["quantized"]
        if sc and (int8 or c < 32):
            raise Rejected(f"layer {i}: shortcut never written")
        if sc and L["activation"] not in (port.LEAKY, port.LINEAR):
            raise Rejected(f"layer {i}: shortcut behind a non-leaky layer")
        if not int8:
            paths[i] = "B" if c < 32 else "A"
    return paths


def run_network_xnor_gpu(layers: Sequence[dict], x: np.ndarray, int8_gpu: bool = False) -> List[Optional[np.ndarray]]:
    """The forward of network_predict_gpu_cudnn (int8_gpu: network_predict_gpu_cudnn_quantized) on an XNOR network: the XNOR
    layers by path A or B, the INT8 layers (int8_gpu and l.quantized) by gpu_rule_oracle, every other layer the oracle's
    CPU function.  Every image is computed as image 0, on its own.  Returns every layer's output over the batch."""
    x = np.ascontiguousarray(x, F32)
    per_image = [_run_image(layers, x[b:b + 1], int8_gpu) for b in range(x.shape[0])]
    return [np.concatenate([pi[i] for pi in per_image], axis=0) for i in range(len(layers))]


def _run_image(layers, x, int8_gpu):
    paths = xnor_paths(layers, int8_gpu)
    outs: List[Optional[np.ndarray]] = []
    cur = np.ascontiguousarray(x, F32)
    folded = {}   # shortcut layer -> the leaky-only value of the XNOR layer in front of it
    for i, l in enumerate(layers):
        t = l["type"]
        if t == port.CONVOLUTIONAL and i in paths:
            if paths[i] == "A":
                o = conv_xnor_a(cur, l)
                if i + 1 < len(layers) and _same_shape_shortcut(layers[i + 1]):
                    folded[i + 1] = conv_xnor_a(cur, l, leaky_only=True)
            else:
                o = conv_xnor_b(cur, l)
        elif t == port.CONVOLUTIONAL and int8_gpu and l["quantized"]:
            o = gro.conv_int8_gpu(cur, l["weights_int8"], l["biases"], l["input_quant_multipler"], l["weights_quant_multipler"],
                                  l["n"], l["size"], l["stride"], l["pad"], l["activation"])
        elif t == port.CONVOLUTIONAL:
            o = port.conv_fp32(cur, l["weights"], l["biases"], l["n"], l["size"], l["stride"], l["pad"], l["activation"])
        elif t == port.SHORTCUT and i in folded:
            o = (outs[l["index"]] + folded[i]).astype(F32)
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
