"""The stems, the input conversion and the small-K XNOR convolutions against the oracle, bit for bit, at their edges.

Five kernel families run only inside whole networks elsewhere: the fused stem + 2x2/2 max-pool + integer input conversion
(k_stem_pool), the 3-channel stem from NCHW (k_conv_stem), the NCHW -> padded-NHWC input conversion (k_input_nchw_to_nhwc),
and the XNOR convolutions with one or two sign words per tap (k_conv_xnor_smallk), alone and with the max-pool and the next
XNOR layer's sign extraction fused in (k_conv_xnor_smallk_pool).  Each case below builds a small network that puts one of
their instantiations to work at an edge: odd pooled sizes, whose last pooled row and column are half outside the image;
channel counts that leave a partial last sign word; filter counts that end in the scalar tail store; the shared-memory limit
of the small-K kernel; one 128-thread block spanning two images (every per-image pixel count is above 128 and not a multiple
of it); and outputs that are channel slices of a [route] buffer, where the 16-byte stores of the stems and of
k_conv_xnor_smallk may run only when the slice starts on a 16-byte boundary.

Each case asserts, through Network.op_kernels, the exact instantiation of every conversion and CUDA-core convolution the
engine launches, and compares each layer with the oracle (oracle/port.py) run on the engine's own input: the fetched output
of the layer in front, or the network input for the stems.  Fused chains are compared at their last layer, whose input
chain the oracle runs layer by layer.  f32 activations must match to the bit, raw XNOR popcounts and INT8 accumulators as
integers.  bf16 networks run on the exactly representable data of test_gpu_tc_exact.py, on which every summation order
gives the same f32 value, and must equal its reference model (run_reference) to the bit; a logistic to within one bf16 ulp.

The helpers and the case table run on the CPU; the tests that need a GPU are marked."""
import numpy as np
import pytest

import exact_model
import ybtest_util as util
from exact_model import Net, consumer_pairs, onehot, run_reference
from ybtest_util import kernel_inst
from yolo2_light_b200 import cfgs

LINEAR, LEAKY, RELU, LOGISTIC = "linear", "leaky", "relu", "logistic"
XNOR = {"xnor": 1, "bin_output": 1}
ACT_CODE = {LEAKY: 7, LINEAR: 3}                                # the ACT_* template argument of k_stem_pool
SMALLK_SMEM = 40 * 1024                                         # conv_kern: n * 9 * CW * 4 bytes of sign words at most


# ---- kernel names -------------------------------------------------------------------------------------------------------
def inst(base, *args):
    """an instantiation: kernel name and template arguments as strings"""
    return base, tuple(str(a) for a in args)


SIMT_F32 = inst("k_conv_simt", "SimtF32")        # any SimtF32 policy
SIMT_XNOR = inst("k_conv_simt", "SimtXnor")


def stem_pool(side, act):
    return inst("k_stem_pool", side, ACT_CODE[act])


def conv_stem(nf, dt):
    return inst("k_conv_stem", nf, "float", "true") if dt == "f32" else inst("k_conv_stem", nf, "bf16", "false")


def smallk(cw):
    return inst("k_conv_xnor_smallk", cw)


def smallk_pool(cw, side):
    return inst("k_conv_xnor_smallk_pool", cw, side)


def nchw(dt):
    return inst("k_input_nchw_to_nhwc", "float" if dt == "f32" else "bf16")


FAMILIES = {
    "k_stem_pool": {stem_pool(s, a) for s in ("SIDE_S8", "SIDE_PM1_S8", "SIDE_BITS") for a in (LEAKY, LINEAR)},
    "k_conv_stem": {conv_stem(nf, dt) for nf in (16, 32) for dt in ("f32", "bf16")},
    "k_input_nchw_to_nhwc": {nchw(dt) for dt in ("f32", "bf16")},
    "k_conv_xnor_smallk": {smallk(cw) for cw in (1, 2)},
    "k_conv_xnor_smallk_pool": {smallk_pool(cw, s) for cw in (1, 2) for s in ("SIDE_PM1_S8", "SIDE_BITS")},
}
TRACKED = set(FAMILIES) | {"k_conv_simt"}        # every launch of these is pinned by the case table

# ---- the case table -----------------------------------------------------------------------------------------------------
class Case:
    """A network on a 3-channel input, the engine's settings, and what it must run and compute:
    kernels  layer -> the one instantiation of a TRACKED kernel that runs it (layer -1: the input conversion); no other
             TRACKED kernel may run
    inputs   layer -> the side format of the one k_int_input op that converts its input
    no_ops   layers with no op of their own (fused into the op in front)
    hidden   layers whose output no op writes: fetch_layer raises
    tc       layer -> its tensor-core plan's kernel
    chains   (first, last): the oracle runs layers first..last from the engine's input of `first`; the engine's layer
             `last` (and, with keep_counts, its raw integer results) must equal it to the bit
    checked  grid-data cases: the layers compared with run_reference"""

    def __init__(self, family, h, w, batch, prec, seed, quantized=False, grid=False):
        self.family, self.prec, self.grid = family, prec, grid
        self.net = Net(3, h, w, batch, seed, calib=[16] * 8 if quantized else None)
        self.q = quantized
        self.fuse, self.keep_counts, self.env = 1, False, {}
        self.kernels, self.inputs, self.no_ops, self.hidden, self.tc, self.chains, self.checked = {}, {}, [], [], {}, [], []

    h = property(lambda self: self.net.h)
    w = property(lambda self: self.net.w)
    batch = property(lambda self: self.net.batch)

    def shapes(self):
        return cfgs.conv_shapes(self.net.secs)

    def conv(self, n, size=3, act=LEAKY, kern="simt", **extra):
        """a convolution with the seeded weights of cfgs.write_weights (sqrt(2 / (k k c)) U(-1, 1), biases U(-0.1, 0.1));
        on grid data, test_gpu_tc_exact's exactly representable ones"""
        if self.grid:
            return self.net.conv(n, size, 1, act, kern, **extra)
        c = self.shapes()[-1]["out_c"] if self.net.n else 3
        rng = self.net.rng
        w = (np.sqrt(2.0 / (size * size * c)) * rng.uniform(-1.0, 1.0, (n, c, size, size))).astype(np.float32)
        b = rng.uniform(-0.1, 0.1, n).astype(np.float32)
        return self.net.conv(n, size, 1, act, kern, w=w, b=b, **extra)

    def maxpool(self):
        return self.net.add("maxpool", size=2, stride=2)

    def images(self, seed):
        if self.grid:     # the stem images of test_gpu_tc_exact: a / 16, a in [0, 16]
            return self.net.images(16, 0, 16)
        return cfgs.synthetic_images(self.batch, 3, self.h, self.w, seed=seed)

    def grid_pixels(self):
        """per-image pixel counts of the launch grids of the kernels under test: the pooled grid of the fused-pool kernels,
        the output of the others, the input of the conversion"""
        s = self.shapes()
        px = [self.h * self.w]
        for j, (base, args) in self.kernels.items():
            if j < 0 or (base, args) == SIMT_F32:
                continue
            k = 1 if base == "k_stem_pool" else j + 1 if base == "k_conv_xnor_smallk_pool" else j
            px.append(s[k]["out_h"] * s[k]["out_w"])
        return px


def c_stem_pool(side, act, h, w, batch, n2=None, xnor_tc=True):
    """(a) stem 3 -> 16, 2x2/2 max-pool, integer layer 2 of C = 16 in side format `side`: one k_stem_pool launch writes
    layer 2's input; with keep_counts layer 2's raw results are checked too"""
    q = side == "SIDE_S8"
    c = Case("stem_pool", h, w, batch, "int", 2000 + h * w + batch, quantized=q)
    c.conv(16, 3, act)
    c.maxpool()
    if q:
        c.conv(24, 3, LEAKY)                     # INT8 (the rule skips linear layers), on the s8 tensor cores
    elif side == "SIDE_PM1_S8":
        c.conv(16, 3, LEAKY, **XNOR)             # +-1 bytes on the s8 tensor cores
    else:
        c.conv(n2, 3, LINEAR, **XNOR)            # sign bits: n < 8, or the tensor cores switched off
        c.kernels[2] = smallk(1)
        if not xnor_tc:
            c.env["YB_XNOR_TC"] = "0"
    c.kernels[0] = stem_pool(side, act)
    c.keep_counts = True
    c.hidden, c.no_ops, c.chains = [0, 1], [1], [(0, 2)]
    return c


def c_conv_stem_f32(nf, act, h, w, batch, then):
    """(b) the f32 stem, in the reference's summation order, where k_stem_pool does not take it"""
    c = Case("conv_stem", h, w, batch, "f32", 2100 + nf + h * w)
    c.conv(nf, 3, act)
    if then == "maxpool":
        c.maxpool()
    else:
        c.conv(8, 3, LEAKY)
        c.kernels[1] = SIMT_F32
    c.kernels[0] = conv_stem(nf, "f32")
    c.chains = [(0, 0)]
    return c


def c_conv_stem_fuse0(h, w, batch):
    """(b) the exact XNOR chain k_stem_pool runs, with fusion off: the stem alone, then max-pool and XNOR layer 2"""
    c = Case("conv_stem", h, w, batch, "int", 2200 + h * w)
    c.conv(16, 3, LEAKY)
    c.maxpool()
    c.conv(16, 3, LEAKY, **XNOR)
    c.fuse = 0
    c.kernels[0] = conv_stem(16, "f32")
    c.chains = [(0, 0), (1, 1), (2, 2)]
    return c


def c_conv_stem_bf16(nf, act, h, w, batch):
    """(c) the bf16 stem of the CUDA cores (YB_NO_STEM_TC), on grid data, with a one-hot consumer on the tensor cores"""
    c = Case("conv_stem", h, w, batch, "bf16", 2300 + nf + h * w, grid=True)
    i = c.conv(nf, 3, act, kern="stem")
    j = c.net.consume()
    if act == LOGISTIC:
        c.net.tol = {i: 1, j: 1}
    c.env["YB_NO_STEM_TC"] = "1"
    c.kernels[0] = conv_stem(nf, "bf16")
    c.checked = [0, 1]
    return c


def c_input(first, dt, h, w, batch):
    """(d) a first layer that is no stem, behind the NCHW -> padded-NHWC conversion: an 8-filter 3x3 convolution, a 16-filter
    1x1 convolution or a max-pool.  f32 on random data; bf16 convolutions on grid data, a bf16 max-pool on the bf16-rounded
    random input (which the conversion makes)."""
    grid = dt == "bf16" and first != "maxpool"
    c = Case("input", h, w, batch, dt, 2400 + len(first) + h * w, grid=grid)
    if first == "maxpool":
        c.maxpool()
    else:
        if first == "conv3x3":
            c.conv(8, 3, LEAKY)
        else:
            c.conv(16, 1, LINEAR)
        c.kernels[0] = SIMT_F32
    c.kernels[-1] = nchw(dt)
    if grid:
        j = c.net.consume()                     # bf16 output: a consumer; 72 filters over 8 channels: CUDA cores
        if c.net.kern[j] == "simt":
            c.kernels[j] = SIMT_F32
        c.checked = [0, j]
    else:
        c.chains = [(0, 0)]
    return c


def c_smallk(C, n, act, h, w, batch, xnor_tc=True):
    """(e) XNOR 3x3/1/1 layer 1 over C channels (CW = ceil(C / 32) sign words per tap) with n filters: k_conv_xnor_smallk
    while its sign words fit the shared memory, else the general popcount kernel"""
    c = Case("smallk", h, w, batch, "int", 2500 + C * 7 + n + h * w)
    c.conv(C, 3, LEAKY)
    c.conv(n, 3, act, **XNOR)
    cw = (C + 31) // 32
    c.kernels.update({-1: nchw("f32"), 0: SIMT_F32, 1: smallk(cw) if n * 9 * cw * 4 <= SMALLK_SMEM else SIMT_XNOR})
    if not xnor_tc:
        c.env["YB_XNOR_TC"] = "0"
    c.keep_counts = True
    c.chains = [(0, 0), (1, 1)]
    return c


def c_smallk_pool(C, n, m, h, w, batch):
    """(f) XNOR layer 1 (C channels, n filters) -> 2x2/2 max-pool -> XNOR layer 3 (n channels, m filters): layer 1's kernel
    writes layer 3's input.  Layer 3 takes +-1 bytes on the tensor cores when n is a multiple of 16 and m >= 8, sign bits on
    k_conv_xnor_smallk otherwise."""
    c = Case("smallk_pool", h, w, batch, "int", 2600 + C + n * 3 + h * w)
    c.conv(C, 3, LEAKY)
    c.conv(n, 3, LEAKY, **XNOR)
    c.maxpool()
    c.conv(m, 3, LINEAR, **XNOR)
    side = "SIDE_PM1_S8" if n % 16 == 0 and m >= 8 else "SIDE_BITS"
    c.kernels.update({-1: nchw("f32"), 0: SIMT_F32, 1: smallk_pool((C + 31) // 32, side)})
    if side == "SIDE_BITS":
        c.kernels[3] = smallk((n + 31) // 32)
    c.hidden, c.no_ops, c.chains = [1, 2], [2], [(0, 0), (1, 3)]
    return c


def c_slice_xnor(coff, h, w, batch):
    """(g) XNOR layer 3 (C = 24, smallk-eligible) writes channels coff.. of route 4's buffer, behind layer 1's coff channels:
    the small-K kernel's float4 stores need a 16-byte aligned slice"""
    c = Case("slice", h, w, batch, "int", 2700 + coff + h * w)
    c.conv(24, 3, LEAKY)                          # 0
    c.conv(coff, 3, LEAKY)                        # 1: first slice of route 4
    c.net.add("route", layers="-2")               # 2: layer 0
    c.conv(16, 3, LEAKY, **XNOR)                  # 3: second slice, at channel coff
    c.net.add("route", layers="1, 3")             # 4
    c.kernels.update({-1: nchw("f32"), 0: SIMT_F32, 1: SIMT_F32, 3: smallk(1) if coff * 4 % 16 == 0 else SIMT_XNOR})
    c.chains = [(0, 0), (1, 1), (3, 3), (4, 4)]
    return c


def c_slice_xnor_input(coff, h, w, batch):
    """(g) XNOR layer 2 (C = 16, a shape the s8 tile takes) reads layer 1, the channel slice at coff of route 3's buffer: the
    tile needs a 16-byte aligned input, so at coff = 6 the layer takes sign bits on k_conv_xnor_smallk"""
    c = Case("slice", h, w, batch, "int", 2900 + coff + h * w)
    c.conv(coff, 3, LEAKY)                        # 0: first slice of route 3
    c.conv(16, 3, LEAKY)                          # 1: second slice, at channel coff
    c.conv(16, 3, LEAKY, **XNOR)                  # 2
    c.net.add("route", layers="0, 1")             # 3
    c.kernels.update({-1: nchw("f32"), 0: SIMT_F32, 1: SIMT_F32, 2: smallk(1)})
    c.inputs[2] = "SIDE_BITS"
    c.chains = [(0, 0), (1, 1), (2, 2), (3, 3)]
    return c


def c_slice_stem(coff, dt, h, w, batch, stem_tc=True):
    """(g) the stem (16 filters) writes channels coff.. of route 2's buffer, behind layer 1's coff channels: unless the slice
    is 16-byte aligned, the stem runs as a plain convolution behind the input conversion.  bf16 on grid data, layer 1 a
    one-hot convolution."""
    c = Case("slice", h, w, batch, dt, 2800 + coff + h * w + stem_tc, grid=dt == "bf16")
    aligned = coff * (4 if dt == "f32" else 2) % 16 == 0
    if dt == "f32":
        c.conv(16, 3, LEAKY)
        c.conv(coff, 3, LEAKY)
        c.chains = [(0, 0), (1, 1), (2, 2)]
    else:
        c.conv(16, 3, LEAKY, kern=("stem" if aligned else "simt"))
        c.net.conv(coff, 3, 1, LINEAR, "reg" if coff >= 8 else "simt", w=onehot(coff, 16, 3, consumer_pairs(16)[:coff]),
                   b=np.zeros(coff, np.float32))
        c.checked = [0, 1, 2]
    c.net.add("route", layers="1, 0")
    if not stem_tc:
        c.env["YB_NO_STEM_TC"] = "1"
    if not aligned:
        c.kernels.update({-1: nchw(dt), 0: SIMT_F32})
    elif dt == "f32" or not stem_tc:
        c.kernels[0] = conv_stem(16, dt)
    else:
        c.tc[0] = "k_stem_tc"
    if dt == "f32" or coff < 8:                   # 8 one-hot bf16 filters run on the tensor cores
        c.kernels[1] = SIMT_F32
    return c


CASES = {
    # (a) k_stem_pool: both sizes odd, one even, a pooled grid 2 pixels high
    "stem_pool_s8_leaky_27x21": lambda: c_stem_pool("SIDE_S8", LEAKY, 27, 21, 3),
    "stem_pool_s8_linear_25x30_b1": lambda: c_stem_pool("SIDE_S8", LINEAR, 25, 30, 1),
    "stem_pool_pm1_leaky_3x263": lambda: c_stem_pool("SIDE_PM1_S8", LEAKY, 3, 263, 3),
    "stem_pool_pm1_linear_21x27": lambda: c_stem_pool("SIDE_PM1_S8", LINEAR, 21, 27, 3),
    "stem_pool_bits_leaky_n6_17x31": lambda: c_stem_pool("SIDE_BITS", LEAKY, 17, 31, 3, n2=6),
    "stem_pool_bits_linear_xnortc0_29x19": lambda: c_stem_pool("SIDE_BITS", LINEAR, 29, 19, 3, n2=16, xnor_tc=False),
    # (b) k_conv_stem<16|32, float, true>
    "stem16_relu_f32_13x11": lambda: c_conv_stem_f32(16, RELU, 13, 11, 3, "maxpool"),
    "stem16_leaky_f32_11x15_b1": lambda: c_conv_stem_f32(16, LEAKY, 11, 15, 1, "maxpool"),
    "stem32_logistic_f32_9x17": lambda: c_conv_stem_f32(32, LOGISTIC, 9, 17, 3, "conv"),
    "stem32_linear_f32_15x13": lambda: c_conv_stem_f32(32, LINEAR, 15, 13, 3, "conv"),
    "stem16_xnor_fuse0_13x11": lambda: c_conv_stem_fuse0(13, 11, 3),
    # (c) k_conv_stem<16|32, bf16>
    "stem16_leaky_bf16_13x11": lambda: c_conv_stem_bf16(16, LEAKY, 13, 11, 3),
    "stem32_linear_bf16_9x17": lambda: c_conv_stem_bf16(32, LINEAR, 9, 17, 3),
    "stem16_relu_bf16_15x13_b1": lambda: c_conv_stem_bf16(16, RELU, 15, 13, 1),
    "stem32_logistic_bf16_11x15": lambda: c_conv_stem_bf16(32, LOGISTIC, 11, 15, 3),
    # (d) k_input_nchw_to_nhwc<float|bf16>
    **{f"input_{first}_{dt}_{h}x{w}{'_b1' if b == 1 else ''}": (lambda first=first, dt=dt, h=h, w=w, b=b: c_input(first, dt, h, w, b))
       for first, dt, h, w, b in [("conv3x3", "f32", 13, 11, 3), ("conv1x1", "f32", 11, 13, 1), ("maxpool", "f32", 15, 9, 3),
                                  ("conv3x3", "bf16", 9, 17, 3), ("conv1x1", "bf16", 11, 15, 1), ("maxpool", "bf16", 13, 11, 3)]},
    # (e) k_conv_xnor_smallk<1|2>, and the general kernel one filter past its shared memory
    **{f"smallk_c{C}_n{n}_{act}{'_xnortc0' if not tc else ''}{'_b1' if b == 1 else ''}":
       (lambda C=C, n=n, act=act, h=h, w=w, b=b, tc=tc: c_smallk(C, n, act, h, w, b, tc))
       for C, n, act, h, w, b, tc in [(8, 1, LEAKY, 13, 11, 3, True), (8, 13, LINEAR, 9, 17, 3, True),
                                      (24, 6, LINEAR, 11, 15, 1, True), (24, 30, LEAKY, 15, 13, 3, True),
                                      (40, 6, LEAKY, 13, 11, 3, True), (40, 13, LINEAR, 17, 9, 3, True),
                                      (56, 1, LINEAR, 9, 19, 3, True), (56, 30, LEAKY, 19, 9, 1, True),
                                      (64, 6, LEAKY, 11, 13, 3, False), (64, 30, LINEAR, 13, 11, 3, False),
                                      (40, 568, LEAKY, 13, 11, 3, True), (40, 569, LEAKY, 13, 11, 3, True)]},
    # (f) k_conv_xnor_smallk_pool<1|2, SIDE_PM1_S8|SIDE_BITS>
    "smallk_pool_cw1_bits_n6_27x21": lambda: c_smallk_pool(24, 6, 8, 27, 21, 3),
    "smallk_pool_cw2_bits_n40_21x27": lambda: c_smallk_pool(40, 40, 8, 21, 27, 3),
    "smallk_pool_cw1_pm1_n16_25x19_b1": lambda: c_smallk_pool(24, 16, 16, 25, 19, 1),
    "smallk_pool_cw2_pm1_n48_23x29": lambda: c_smallk_pool(56, 48, 24, 23, 29, 3),
    # (g) route slices
    "slice_xnor_at6_13x11": lambda: c_slice_xnor(6, 13, 11, 3),
    "slice_xnor_at4_11x13_b1": lambda: c_slice_xnor(4, 11, 13, 1),
    "slice_xnor_input_at6_13x11": lambda: c_slice_xnor_input(6, 13, 11, 3),
    "slice_stem_at6_f32_13x11": lambda: c_slice_stem(6, "f32", 13, 11, 3),
    "slice_stem_at8_f32_11x15_b1": lambda: c_slice_stem(8, "f32", 11, 15, 1),
    "slice_stem_at6_bf16_13x11": lambda: c_slice_stem(6, "bf16", 13, 11, 3),
    "slice_stem_at8_bf16_9x17": lambda: c_slice_stem(8, "bf16", 9, 17, 3),
    "slice_stem_at8_bf16_nostemtc_15x13": lambda: c_slice_stem(8, "bf16", 15, 13, 3, stem_tc=False),
}


# ---- CPU tests ----------------------------------------------------------------------------------------------------------
KERNEL_NAMES = [   # (name as cudaFuncGetName gives it -- nvcc's mangling, as in ptxas -v --, its c++filt form, instantiation)
    ("_ZN2yb11k_stem_poolILNS_7SideFmtE2ELi7EEEvPKfNS_2TVENS_5StemWILi16EEEiiif",
     "void yb::k_stem_pool<(yb::SideFmt)2, 7>(float const*, yb::TV, yb::StemW<16>, int, int, int, float)",
     stem_pool("SIDE_S8", LEAKY)),
    ("_ZN2yb11k_conv_stemILi32E13__nv_bfloat16Lb0EEEvPKfNS_2TVENS_5StemWIXT_EEEiii",
     "void yb::k_conv_stem<32, __nv_bfloat16, false>(float const*, yb::TV, yb::StemW<32>, int, int, int)", conv_stem(32, "bf16")),
    ("_ZN2yb11k_conv_stemILi16EfLb1EEEvPKfNS_2TVENS_5StemWIXT_EEEiii",
     "void yb::k_conv_stem<16, float, true>(float const*, yb::TV, yb::StemW<16>, int, int, int)", conv_stem(16, "f32")),
    ("_ZN2yb23k_conv_xnor_smallk_poolILi2ELNS_7SideFmtE4EEEvNS_5XnorPENS_2TVE",
     "void yb::k_conv_xnor_smallk_pool<2, (yb::SideFmt)4>(yb::XnorP, yb::TV)", smallk_pool(2, "SIDE_BITS")),
    ("_ZN2yb18k_conv_xnor_smallkILi1EEEvNS_5XnorPE", "void yb::k_conv_xnor_smallk<1>(yb::XnorP)", smallk(1)),
    ("_ZN2yb20k_input_nchw_to_nhwcI13__nv_bfloat16EEvPKfNS_2TVE",
     "void yb::k_input_nchw_to_nhwc<__nv_bfloat16>(float const*, yb::TV)", nchw("bf16")),
    ("_ZN2yb11k_conv_simtINS_8SimtXnorEEEvNS_5SimtPE", "void yb::k_conv_simt<yb::SimtXnor>(yb::SimtP)", SIMT_XNOR),
    ("_ZN2yb11k_conv_simtINS_7SimtF32I13__nv_bfloat16S2_fLb0EEEEEvNS_5SimtPE",
     "void yb::k_conv_simt<yb::SimtF32<__nv_bfloat16, __nv_bfloat16, float, false> >(yb::SimtP)", SIMT_F32),
    ("_ZN2yb9k_maxpoolIfEEvNS_2TVES1_iii", "void yb::k_maxpool<float>(yb::TV, yb::TV, int, int, int)", inst("k_maxpool", "float")),
]


@pytest.mark.parametrize("mangled,demangled,expected", KERNEL_NAMES)
def test_kernel_inst(mangled, demangled, expected):
    assert kernel_inst(mangled) == expected
    assert kernel_inst(demangled) == expected


def test_every_instantiation_has_a_case():
    ran = {k for name in CASES for k in CASES[name]().kernels.values()}
    for fam, insts in FAMILIES.items():
        assert insts <= ran, (fam, insts - ran)
    assert SIMT_XNOR in ran


def test_every_family_has_a_batch_1_case():
    fams = {CASES[name]().family for name in CASES}
    for fam in fams:
        assert any(CASES[n]().family == fam and CASES[n]().batch == 1 for n in CASES), fam
        assert any(CASES[n]().family == fam and CASES[n]().batch == 3 for n in CASES), fam


def test_fused_pool_cases_have_odd_sizes():
    """every fused-pool case pools an output with an odd height or width: its last pooled row or column is half outside"""
    n = 0
    for name in CASES:
        c = CASES[name]()
        s = c.shapes()
        for j, (base, _) in c.kernels.items():
            if base in ("k_stem_pool", "k_conv_xnor_smallk_pool"):
                assert s[j]["out_h"] % 2 or s[j]["out_w"] % 2, name
                n += 1
    assert n == 10


def test_smallk_cases_have_partial_words_or_a_scalar_tail():
    for name in CASES:
        c = CASES[name]()
        s = c.shapes()
        for j, (base, _) in c.kernels.items():
            if base in ("k_conv_xnor_smallk", "k_conv_xnor_smallk_pool"):
                assert s[j]["c"] % 32 != 0 or s[j]["n"] % 4 != 0, (name, j)


def test_shared_memory_edge():
    """n = 568 sign-word filters of CW = 2 fill the small-K kernel's shared memory, n = 569 do not"""
    assert 568 * 9 * 2 * 4 <= SMALLK_SMEM < 569 * 9 * 2 * 4
    assert CASES["smallk_c40_n568_leaky"]().kernels[1] == smallk(2)
    assert CASES["smallk_c40_n569_leaky"]().kernels[1] == SIMT_XNOR


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_shapes(name):
    """non-square odd inputs at batch 1 or 3, and launch grids where one 128-thread block spans two images"""
    c = CASES[name]()
    assert c.h != c.w and (c.h % 2 or c.w % 2) and c.batch in (1, 3), name
    for px in c.grid_pixels():
        assert px > 128 and px % 128 != 0, (name, px)
    s = c.shapes()
    for j in list(c.kernels) + c.no_ops + c.hidden + list(c.tc):
        assert -1 <= j < len(s), (name, j)
    for j, (base, _) in c.kernels.items():
        if base in ("k_stem_pool", "k_conv_stem"):
            assert j == 0 and s[0]["type"] == "convolutional" and s[0]["c"] == 3 and s[0]["n"] in (16, 32), name
        elif base in ("k_conv_xnor_smallk", "k_conv_xnor_smallk_pool"):
            assert s[j]["xnor"] and s[j]["size"] == 3 and s[j]["c"] <= 64, name


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n]().grid))
def test_grid_case_premise(name):
    """the grid-data cases are exact in any summation order"""
    c = CASES[name]()
    x = c.images(0)
    _, units = run_reference(c.net, x, adt_bf16=True)
    assert units and max(units.values()) < 2 ** 20


# ---- GPU tests ----------------------------------------------------------------------------------------------------------
def check_chains(case, m, x):
    q, bf16 = case.q, case.prec == "bf16"
    layers = m.layers
    for first, last in case.chains:
        if layers[last]["type_name"] == "ROUTE":
            exp, cnt = np.concatenate([m.fetch_layer(int(j), quantized=q) for j in layers[last]["input_layers"]], axis=1), None
        else:
            cur = (util.bf16_round(x) if bf16 else x) if first == 0 else m.fetch_layer(first - 1, quantized=q)
            for i in range(first, last + 1):
                cur, cnt = util.oracle_layer(layers[i], i, cur, int(q))
            exp = util.bf16_round(cur) if bf16 else cur
        got = m.fetch_layer(last, quantized=q)
        bad = np.argwhere(got.view(np.uint32) != np.ascontiguousarray(exp, np.float32).view(np.uint32))
        assert got.shape == exp.shape and len(bad) == 0, (first, last, len(bad), bad[:5].tolist())
        if case.keep_counts and cnt is not None:
            assert np.array_equal(m.fetch_counts(last, quantized=q), cnt), (first, last)


def check_grid(case, m, x):
    exp, _ = run_reference(case.net, x, adt_bf16=True)
    for i in case.checked:
        got = m.fetch_layer(i).transpose(0, 2, 3, 1)
        e = np.ascontiguousarray(exp[i])
        assert got.shape == e.shape, i
        tol = case.net.tol.get(i, 0)
        if tol:
            d = util.ulp_diff(got, e, True)
            assert np.all(got >= 0) and np.all(e >= 0) and np.array_equal(np.signbit(got), np.signbit(e)) and d.max() <= tol, \
                (i, int(d.max()))
        else:
            bad = np.argwhere(got.view(np.uint32) != e.view(np.uint32))
            assert len(bad) == 0, (i, len(bad), bad[:5].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_stem_xnor(name, workdir, monkeypatch):
    import yolo2_light_b200 as yb
    case = CASES[name]()
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    m = util.load(*exact_model.write_net(case.net, workdir, f"sx_{name}"), case.batch, quantized=int(case.q),
                  precision=yb.YB_PREC_FP32 if case.prec == "f32" else yb.YB_PREC_BF16_TC, fuse=case.fuse,
                  keep_counts=case.keep_counts)
    q = case.q
    ops = m.op_kernels(quantized=q)
    ran = {}
    for j, _, k in ops:
        if k is not None and any(b in k for b in TRACKED) and kernel_inst(k)[0] in TRACKED:
            ran.setdefault(j, []).append(kernel_inst(k))
    assert ran == {j: [k] for j, k in case.kernels.items()}, (name, ran)
    for j, side in case.inputs.items():
        conv = [kernel_inst(k) for jj, _, k in ops if jj == j and util.kernel_is(k, "k_int_input")]
        assert conv == [inst("k_int_input", side)], (name, j, conv)
    for j in case.no_ops:
        assert not [op for op in ops if op[0] == j], (name, j, ops)
    for j, kern in case.tc.items():
        assert m.tc_plan(j, quantized=q).get("kernel") == kern, (name, j, m.tc_plan(j, quantized=q))
    x = case.images(seed=sum(map(ord, name)))
    m.predict(x, quantized=q)
    for j in case.hidden:
        with pytest.raises(yb.YbError):
            m.fetch_layer(j, quantized=q)
    if case.grid:
        check_grid(case, m, x)
    else:
        check_chains(case, m, x)
    if case.family == "smallk_pool":    # unfused: the same bits
        last = case.chains[-1][1]
        fused = m.fetch_layer(last, quantized=q).copy()
        m.set_option("fuse", 0)
        m.predict(x, quantized=q)
        assert util.bits_equal(m.fetch_layer(last, quantized=q), fused), name
