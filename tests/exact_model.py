"""The exact-data model of the tensor-core convolution tests: data on which every convolution is exact, the networks built
on it, and a host model of the engine that gives every layer's output to the bit.

Activations are a/8 (a in [-8, 8]; stem images a/16, a in [0, 16]), weights b/64 (b in [-8, 8]), biases c/512.  Every
product is then exact in bf16 / tf32, every partial sum a multiple of the product grid, and while sum |x| |w| over a dot
product stays below 2^20 grid units every partial sum is an exact f32 number in any summation order, whatever the tensor
core's alignment of its addends and with or without FMA contraction.  The accumulator is the float64 dot product; the
epilogue is a few IEEE f32 operations (bias add, leaky, residual add, second leaky, round to bf16) that numpy float32
repeats bit for bit.  `premise` checks these conditions on the host for every convolution before anything runs.

Under the GPU INT8 rule (`quantized` = 2) the activations stay f32 and the float convolutions take the tf32 wgmma: grid
data is exact in tf32 as well, so those layers are bit for bit too.  A layer behind one reads f32 values off the tf32 grid
(leaky outputs); only one-hot consumers do, and `tf32_round` gives what they see."""
import hashlib
import struct

import numpy as np

import ybtest_util as util
from ybtest_util import bf16_round
from yolo2_light_b200 import cfgs

LINEAR, LEAKY, RELU, LOGISTIC = "linear", "leaky", "relu", "logistic"
BOUND_UNITS = 2 ** 20          # |partial sums| in product-grid units: 4 bits below f32's 24-bit significand
F32_01 = np.float32(0.1)


# ---- data ---------------------------------------------------------------------------------------------------------------
def grid_acts(rng, shape, den=8, lo=-8, hi=8):
    return (rng.integers(lo, hi + 1, shape) / den).astype(np.float32)


def grid_weights(rng, n, c, k):
    return (rng.integers(-8, 9, (n, c, k, k)) / 64).astype(np.float32)


def grid_bias(rng, n, den=512, lim=512):
    return (rng.integers(-lim, lim + 1, n) / den).astype(np.float32)


def onehot(n, c, k, pairs):
    """n filters, filter j reads channel pairs[j][0] through tap pairs[j][1] (ky * k + kx) with weight 1"""
    w = np.zeros((n, c, k, k), np.float32)
    for j, (ch, t) in enumerate(pairs):
        w[j, ch, t // k, t % k] = 1.0
    return w


def consumer_pairs(c):
    """(channel, tap) of every filter of a one-hot 3x3 consumer over c channels: all 9 taps of every channel (9 c filters)"""
    return [(j % c, (j // c + j % c) % 9) for j in range(9 * c)]


class Net:
    """A small network under construction: cfg sections, the weights of each convolution and what each is expected to
    run on ("reg" k_conv_tc_reg, "tc" k_conv_tc, "stem" k_stem_tc, "stem_s2" k_stem_s2_tc, "s8_gpu" the GPU rule's INT8
    tile, "simt" the CUDA cores).  `quantized` is the flag the cfg is parsed with, `rule` the INT8 rule it runs under: a
    rule-2 network parsed with 0 has no INT8 layer, and every float convolution with a reader takes tf32."""

    def __init__(self, c, h, w, batch, seed, calib=None, rule=0):
        net = cfgs._net(w, h, calib)
        net[1]["channels"] = str(c)
        self.secs = [net]
        self.rng = np.random.default_rng(seed)
        self.batch, self.c, self.h, self.w = batch, c, h, w
        self.params = {}     # layer -> (weights [n][c][k][k], bias)
        self.kern = {}       # layer -> expected kernel
        self.edges = []      # (layer, description, predicate on the plan)
        self.env = {}
        self.quantized = 0
        self.rule = rule
        self.fuse = 1
        self.x = None        # the input images, when a case sets them
        self.tol = {}        # layer -> bf16 ulps its output may differ by (the double-precision logistic), else 0

    @property
    def n(self):
        return len(self.secs) - 1

    def shapes(self):
        return cfgs.conv_shapes(self.secs)

    def conv(self, n, size=3, stride=1, act=LEAKY, kern=None, w=None, b=None, **extra):
        """kern None: the tensor-core kernel of a float layer with a reader, k_conv_tc_reg (bf16) or k_conv_tc (tf32)"""
        kern = kern or ("tc" if self.rule == 2 else "reg")
        self.secs.append(cfgs._conv(n, size, stride, bn=False, act=act, **extra))
        c = self.shapes()[-1]["c"]
        w = grid_weights(self.rng, n, c, size) if w is None else w
        b = grid_bias(self.rng, n) if b is None else b
        i = self.n - 1
        self.params[i] = (np.asarray(w, np.float32), np.asarray(b, np.float32))
        self.kern[i] = kern
        return i

    def preserve(self, kern=None):
        """grid-preserving 1x1 layer: one-hot weights over a permutation of the channels, a bias on the activation grid,
        linear -- its output stays exactly on the activation grid"""
        c = self.shapes()[-1]["out_c"] if self.n else self.c
        perm = self.rng.permutation(c)
        w = onehot(c, c, 1, [(int(perm[j]), 0) for j in range(c)])
        return self.conv(c, 1, 1, LINEAR, kern, w=w, b=grid_acts(self.rng, c, 8, -4, 4))

    def consume(self):
        """one-hot 3x3 consumer of the last layer's output (f32 out when it is the last layer): k_conv_tc where its channels
        fill whole 32-byte rows (16 bf16, 8 tf32 channels), else the CUDA cores.  Under rule 2 a convolution without a
        reader runs on the CUDA cores, so a tf32 consumer is read by a [route] alias."""
        c = self.shapes()[-1]["out_c"]
        pairs = consumer_pairs(c)
        kern = "tc" if c % (8 if self.rule == 2 else 16) == 0 else "simt"
        i = self.conv(len(pairs), 3, 1, LINEAR, kern, w=onehot(len(pairs), c, 3, pairs), b=np.zeros(len(pairs), np.float32))
        if self.rule == 2 and kern == "tc":
            self.add("route", layers="-1")
        return i

    def add(self, name, **opts):
        self.secs.append((name, {k: str(v) for k, v in opts.items()}))
        return self.n - 1

    def edge(self, layer, what, pred):
        self.edges.append((layer, what, pred))
        return self

    def images(self, den=8, lo=-8, hi=8):
        return grid_acts(np.random.default_rng(self.rng.integers(1 << 30)), (self.batch, self.c, self.h, self.w), den, lo, hi)


def write_weights(net, path):
    """The convolutions' weights in the reference's .weights format (cfgs.write_weights), no batch norm: biases[n], then
    weights[n][c][k][k] per convolution in cfg order"""
    with open(path, "wb") as f:
        f.write(struct.pack("<iiiQ", 0, 2, 0, 0))
        for i in sorted(net.params):
            w, b = net.params[i]
            b.astype("<f4").tofile(f)
            w.astype("<f4").tofile(f)
    return path


def write_net(net, workdir, name):
    """the network's cfg and grid-data weights through ybtest_util.write_net, the weights' digest standing for the seed"""
    h = hashlib.sha1()
    for i in sorted(net.params):
        for a in net.params[i]:
            h.update(a.tobytes())
    return util.write_net(workdir, name, net.secs, h.hexdigest(), weights=lambda path: write_weights(net, path))


# ---- reference ----------------------------------------------------------------------------------------------------------
def conv_acc(x, w, stride, pad):
    """float64 accumulators of a convolution over NHWC x: one matmul per tap"""
    x = np.asarray(x, np.float64)
    B, H, W, C = x.shape
    n, _, k, _ = w.shape
    OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    xp = np.zeros((B, H + 2 * pad, W + 2 * pad, C))
    xp[:, pad:pad + H, pad:pad + W] = x
    acc = np.zeros((B, OH, OW, n))
    w = np.asarray(w, np.float64)
    for ky in range(k):
        for kx in range(k):
            xs = xp[:, ky:ky + stride * (OH - 1) + 1:stride, kx:kx + stride * (OW - 1) + 1:stride, :]
            acc += xs @ w[:, :, ky, kx].T
    return acc


def grid_step(a):
    """the coarsest power of two 2^-e (e <= 40) of which every element of a is a multiple"""
    a = np.asarray(a, np.float64)
    for e in range(41):
        s = a * 2.0 ** e
        if np.array_equal(s, np.round(s)):
            return 2.0 ** -e
    raise AssertionError("data off every binary grid")


def premise(x, w, b, stride, pad):
    """every partial sum of the convolution, and the bias add, is exact in f32 in any order; returns the largest
    sum |x| |w| + |b| in units of the grid of those sums (0 for one-hot filters)"""
    nz = w != 0
    if np.all(nz.reshape(len(w), -1).sum(1) <= 1) and np.all(np.abs(w[nz]) == 1):
        # one-hot filters: a single product per output, then the bias add, which must be exact itself
        acc = conv_acc(x, w, stride, pad) + 0.0
        s = acc.astype(np.float32) + b.astype(np.float32)
        assert np.array_equal(s.astype(np.float64), acc + np.asarray(b, np.float64)), "one-hot layer: bias add rounds"
        return 0.0
    g = min(grid_step(x) * grid_step(w), grid_step(b))     # every partial sum and the bias add are multiples of g
    units = (conv_acc(np.abs(x), np.abs(w), stride, pad) + np.abs(b)).max() / g
    assert units < BOUND_UNITS, f"sum |x||w| = {units:.3g} grid units >= 2^20"
    return units


def leaky_tc(a):
    """fmaxf(a, 0.1f * a): the epilogues of k_conv_tc_reg, k_conv_tc, k_stem_tc and k_stem_s2_tc"""
    return np.maximum(a, F32_01 * a)


def leaky_exact(a):
    """act_exact: a > 0 ? a : (float)(0.1 * (double)a), the CUDA-core kernels (the reference's activate())"""
    return np.where(a > 0, a, (0.1 * a.astype(np.float64)).astype(np.float32)).astype(np.float32)


def activate(a, act, kern):
    """the epilogue's activation: leaky as leaky_exact on the CUDA cores and leaky_tc on the tensor cores; relu and logistic
    only run on the CUDA cores (act_exact): x * (x > 0), which is -0 for x < 0, and (float)(1 / (1 + exp(-(double)x))), which
    numpy's float64 exp reproduces to within one f32 ulp"""
    if act == LEAKY:
        return leaky_exact(a) if kern == "simt" else leaky_tc(a)
    if act == RELU:
        return a * (a > 0)
    if act == LOGISTIC:
        return (1.0 / (1.0 + np.exp(-a.astype(np.float64)))).astype(np.float32)
    assert act == LINEAR, act
    return a


def epilogue(acc, b, act, kern, res=None, act2=LINEAR, bf16=True):
    a = activate((acc + 0.0).astype(np.float32) + b.astype(np.float32), act, kern)
    if res is not None:
        a = activate(a + res.astype(np.float32), act2, kern)
    return bf16_round(a) if bf16 else a.astype(np.float32)


def run_reference(net, x, adt_bf16=True):
    """Host model of the engine on these networks: every layer's output as stored (NHWC f32 values; bf16-rounded where the
    engine keeps bf16), the [yolo] layers' raw head values, and the premise of every convolution.  Follows the engine's
    layer plan: bf16 outputs unless a convolution has no consumer or only detection layers read it; conv + same-shape
    shortcut fused when `fuse` is on, the conv is stride 1 and the shortcut its sole reader.  An INT8 layer ("s8_gpu") is
    not modelled: its output is None, and the test checks it against the oracle on its fetched input.  A tf32 consumer's
    output is the copy of its input at full f32 precision, which the test replaces with tf32_round's."""
    shapes = net.shapes()
    secs = net.secs[1:]
    cons = {i: [] for i in range(len(secs))}
    for i, L in enumerate(shapes):
        t = L["type"]
        if t == "route":
            for j in L["layers"]:
                cons[j].append(i)
        elif t == "shortcut":
            cons[i - 1].append(i); cons[L["index"]].append(i)
        elif i > 0:
            cons[i - 1].append(i)
    outs, units = {}, {}
    cur = np.ascontiguousarray(x.transpose(0, 2, 3, 1))
    if net.kern.get(0, "").startswith("stem"):
        cur = bf16_round(cur) if adt_bf16 else cur
    fused_res = {}
    for i, L in enumerate(shapes):
        t = L["type"]
        if t == "convolutional":
            if net.kern[i] == "s8_gpu":
                outs[i] = cur = None
                continue
            w, b = net.params[i]
            units[i] = premise(cur, w, b, L["stride"], L["pad"])
            acc = conv_acc(cur, w, L["stride"], L["pad"])
            heads_only = bool(cons[i]) and all(shapes[r]["type"] in ("yolo", "region") for r in cons[i])
            bf16 = adt_bf16 and bool(cons[i]) and not heads_only
            nxt = shapes[i + 1] if i + 1 < len(shapes) else None
            if (net.fuse and nxt is not None and nxt["type"] == "shortcut" and cons[i] == [i + 1] and L["stride"] == 1
                    and nxt["index"] != i):
                fused_res[i + 1] = (acc, b, L["activation"], net.kern[i])
                outs[i] = None
                continue
            cur = epilogue(acc, b, L["activation"], net.kern[i], bf16=bf16)
        elif t == "shortcut":
            res = outs[L["index"]]
            act2 = secs[i][1].get("activation", LINEAR)
            if i in fused_res:
                acc, b, act, kern = fused_res[i]
                cur = epilogue(acc, b, act, kern, res=res, act2=act2, bf16=adt_bf16)
            else:
                a = cur + res
                cur = leaky_exact(a) if act2 == LEAKY else a
                cur = bf16_round(cur) if adt_bf16 else cur
        elif t == "route":
            cur = np.concatenate([outs[j] for j in L["layers"]], axis=3)
        elif t == "yolo":
            pass   # the head's f32 values stay in `cur`; the test applies the logistic
        else:
            raise NotImplementedError(t)
        outs[i] = cur
    return outs, units


def tf32_round(a, mode):
    """f32 values as a tf32 operand: "rz" drops the 13 low significand bits, "rn" rounds to nearest even, "rna" to nearest
    with ties away from zero (cvt.rna.tf32.f32).  The PTX ISA does not say which one the tf32 wgmma applies to f32 operands."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    if mode == "rn":
        u = u + 0xFFF + ((u >> 13) & 1)
    elif mode == "rna":
        u = u + 0x1000
    else:
        assert mode == "rz", mode
    return ((u >> 13) << 13 & 0xFFFFFFFF).astype(np.uint32).view(np.float32).reshape(np.shape(a))


def shifted_copies(t, pairs):
    """the one-hot 3x3 consumer's output: filter j = t[..., c_j] shifted by tap t_j, zero border (NHWC); + 0 as the
    consumer's accumulator, which starts at +0 and so turns a -0 input (relu) into +0"""
    B, H, W, C = t.shape
    tp = np.zeros((B, H + 2, W + 2, C), np.float32)
    tp[:, 1:H + 1, 1:W + 1] = t + np.float32(0)
    return np.stack([tp[:, tap // 3:tap // 3 + H, tap % 3:tap % 3 + W, c] for c, tap in pairs], axis=3)
