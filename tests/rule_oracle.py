"""CPU restatement of the reference's integer and XNOR rules, for the tests: which arithmetic each convolution gets under an INT8
rule (`quantized` 0, 1 or 2) and an XNOR rule (conv_arith, named as the engine's Arith), the GPU build's conversions and
convolutions, and the whole forward (forward) on port.run_network's layer loop.

The GPU INT8 mode (network_predict_gpu_cudnn_quantized, yolov2_forward_network_gpu.cu:576) follows
forward_network_gpu_cudnn_quantized's loop (:494-507); the GPU build's XNOR arithmetic is forward_convolutional_layer_gpu_cudnn
(:23-139).  Everything is numpy in IEEE float32 / exact integers, so each value is defined bit for bit:
  int8_gpu    conversion v = x * m rounded once in float32; CUDA's float -> int (truncation, saturating at +-2^31, NaN -> 0);
              clamp to +-127 (cuda_f32_to_int8 + max_abs, gpu.cu:730-739).  v <= -2^31 gives -127: max_abs read without
              overflow; what the reference binary does with abs(INT_MIN) depends on its compiler.
              convolution acc = sum wq * xq over the in-image taps, exact (float64 products and sums of s8 values stay below
              2^53); y = (float)acc * ALPHA1, ALPHA1 = 1 / (m_in * m_w) (:200); y += bias; then activate() of the scalar build
              (additionally.h:85-91) -- one rounded multiply and one rounded add.
  xnor_gpu    (path A) c % 32 == 0, any geometry: input bit x > 0, out-of-image taps -1, dot = 2*count - K (exact);
              y = fmaf((float)dot, mean, bias), correctly rounded once (fmaf_f32 below); leaky `y >= 0 ? y : 0.1f*y` in float,
              any other activation after it.  A same-shape [shortcut] behind it is `from + v`, v the leaky-only value, with no
              activation.
  pm1z_gpu    (path B) c < 32: s = sum sign(w) * (x >= 0 ? +1 : -1), out-of-image taps 0 (exact); y = act((float)s * mean + bias)
              with a rounded multiply and a rounded add.
  act         leaky in float (0.1f * y), logistic in double as every other layer of the engine, relu and linear exact.
"""
from fractions import Fraction
from typing import List, Optional, Sequence

import numpy as np

from oracle import port

F32 = np.float32
XNOR_CPU, XNOR_GPU = 0, 1      # yb.YB_XNOR_CPU, yb.YB_XNOR_GPU


class Rejected(ValueError):
    """A network the GPU XNOR rule does not run."""


# ---- the GPU INT8 rule --------------------------------------------------------------------------------------------------
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


def _cols(xp, size, stride, oh, ow):
    c = xp.shape[0]
    cols = np.empty((c, size, size, oh, ow), np.float64)   # K ordered (c, ky, kx), the weights' order
    for ky in range(size):
        for kx in range(size):
            cols[:, ky, kx] = xp[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride]
    return cols.reshape(c * size * size, oh * ow)


def conv_int8_gpu(x, weights_int8, biases, input_mult, weights_mult, n, size, stride, pad, activation, want_acc=False):
    x = np.asarray(x, F32)
    b, c, h, w = x.shape
    oh, ow = (h + 2 * pad - size) // stride + 1, (w + 2 * pad - size) // stride + 1
    wq = np.asarray(weights_int8, np.int8).reshape(n, c * size * size).astype(np.float64)
    acc = np.empty((b, n, oh, ow), np.int32)
    for k in range(b):
        xq = np.pad(quantize_input_gpu(x[k], input_mult).astype(np.float64), ((0, 0), (pad, pad), (pad, pad)))
        acc[k] = (wq @ _cols(xq, size, stride, oh, ow)).astype(np.int64).reshape(n, oh, ow)
    alpha1 = F32(1) / (F32(input_mult) * F32(weights_mult))
    y = acc.astype(F32) * alpha1
    y = y + np.asarray(biases, F32).reshape(1, n, 1, 1)
    out = activate(y, activation)
    return (out, acc) if want_acc else out


# ---- the GPU XNOR rule --------------------------------------------------------------------------------------------------
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
    return activate(y, act)


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


# ---- the rules ----------------------------------------------------------------------------------------------------------
def conv_arith(layers: Sequence[dict], i: int, quantized: int = 0, xnor_rule: int = XNOR_CPU) -> str:
    """The arithmetic of convolution i: "f32", "xnor_pm1_f32" (the CPU XNOR rule's float fallback at stride != 1 or pad != 1),
    "xnor", "xnor_gpu" (path A), "pm1z_gpu" (path B), "int8" or "int8_gpu".  INT8 takes precedence over XNOR under both rules:
    the CPU rule's every non-linear layer but the first, the GPU rule's l.quantized.  Raises Rejected for an XNOR layer the GPU
    XNOR rule does not run."""
    L = layers[i]
    if quantized == 1 and i >= 1 and L["activation"] != port.LINEAR:
        return "int8"
    int8 = quantized == 2 and bool(L["quantized"])
    if xnor_rule == XNOR_GPU and L["xnor"]:
        sc = i + 1 < len(layers) and _same_shape_shortcut(layers[i + 1])
        c = L["c"]
        if c >= 32 and c % 32:
            raise Rejected(f"layer {i}: c = {c}")
        if sc and (int8 or c < 32):
            raise Rejected(f"layer {i}: shortcut never written")
        if sc and L["activation"] not in (port.LEAKY, port.LINEAR):
            raise Rejected(f"layer {i}: shortcut behind a non-leaky layer")
    if int8:
        return "int8_gpu"
    if not L["xnor"]:
        return "f32"
    if xnor_rule == XNOR_GPU:
        return "pm1z_gpu" if L["c"] < 32 else "xnor_gpu"
    return "xnor" if L["stride"] == 1 and L["pad"] == 1 else "xnor_pm1_f32"


def conv(L: dict, arith: str, x: np.ndarray, want_raw: bool = False):
    """Convolution L under `arith` on x; want_raw: (output, the raw XNOR popcounts, dot or s, or the INT8 accumulators; None
    for "f32").  The CPU XNOR rule's two arithmetics are the oracle's XNOR convolution."""
    if arith == "int8":
        return port.conv_int8(x, L["weights_int8"], L["biases"], L["input_quant_multipler"], L["weights_quant_multipler"],
                              L["n"], L["size"], L["stride"], L["pad"], L["activation"], want_acc=want_raw)
    if arith == "int8_gpu":
        return conv_int8_gpu(x, L["weights_int8"], L["biases"], L["input_quant_multipler"], L["weights_quant_multipler"],
                             L["n"], L["size"], L["stride"], L["pad"], L["activation"], want_acc=want_raw)
    if arith == "xnor_gpu":
        return conv_xnor_a(x, L, want_raw=want_raw)
    if arith == "pm1z_gpu":
        return conv_xnor_b(x, L, want_raw=want_raw)
    if arith in ("xnor", "xnor_pm1_f32"):
        return port.conv_xnor(x, L["weights"], L["biases"], L["mean_arr"], L["n"], L["size"], L["activation"],
                              want_counts=want_raw)
    out = port.conv_fp32(x, L["weights"], L["biases"], L["n"], L["size"], L["stride"], L["pad"], L["activation"])
    return (out, None) if want_raw else out


def forward(layers: Sequence[dict], x: np.ndarray, quantized: int = 0, xnor_rule: int = XNOR_CPU) -> List[Optional[np.ndarray]]:
    """Every layer's output of the reference's forward under the INT8 rule `quantized` (0 none, 1 the CPU build's, 2 the GPU
    build's) and the XNOR rule: port.run_network's layer loop with each convolution in its conv_arith.  Under the GPU XNOR
    rule a same-shape [shortcut] behind a path-A layer is the bit GEMM's `from + v`, and every image is computed as image 0,
    on its own."""
    x = np.ascontiguousarray(x, F32)
    if xnor_rule == XNOR_GPU and x.shape[0] > 1:
        per_image = [forward(layers, x[b:b + 1], quantized, xnor_rule) for b in range(x.shape[0])]
        return [np.concatenate([pi[i] for pi in per_image], axis=0) for i in range(len(layers))]
    folded = {}   # shortcut layer -> the leaky-only value of the path-A layer in front of it

    def layer_fn(i, L, cur, outs):
        if L["type"] == port.CONVOLUTIONAL:
            arith = conv_arith(layers, i, quantized, xnor_rule)
            if arith == "xnor_gpu" and i + 1 < len(layers) and _same_shape_shortcut(layers[i + 1]):
                folded[i + 1] = conv_xnor_a(cur, L, leaky_only=True)
            return conv(L, arith, cur)
        if i in folded:
            return (outs[L["index"]] + folded[i]).astype(F32)
        return None

    return port.run_network(layers, x, layer_fn=layer_fn)
