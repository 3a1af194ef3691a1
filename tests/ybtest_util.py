"""Shared helpers for the test-suite: small model zoo (generated cfg + seeded weights), reference/oracle access."""
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from yolo2_light_b200 import cfgs  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

def edge_shapes_yolo(width=40, height=24):
    """Shortcuts across shapes (from 2x and 4x larger, from half the size, from fewer and more channels), upsamples with
    scale != 1, an explicitly padded 3/2 max-pool and a one-class [yolo] head, on a non-square input."""
    mp = lambda size, stride, padding: ("maxpool", {"size": str(size), "stride": str(stride), "padding": str(padding)})
    sc = lambda frm, act: ("shortcut", {"from": str(frm), "activation": act})
    return [cfgs._net(width, height),
            cfgs._conv(8, 3),                                        # 0: H x W x 8
            cfgs._conv(8, 3, 2),                                     # 1: H/2
            sc(0, "linear"),                                         # 2: from 2x larger
            cfgs._conv(12, 3, 2),                                    # 3: H/4 x 12
            sc(0, "leaky"),                                          # 4: from 4x larger, 8 of 12 channels
            ("upsample", {"stride": "2", "scale": "0.5"}),           # 5: H/2 x 12
            sc(3, "relu"),                                           # 6: from half the size
            cfgs._conv(6, 1),                                        # 7: H/2 x 6
            sc(5, "logistic"),                                       # 8: from 12 channels onto 6
            ("upsample", {"stride": "3", "scale": "1.5"}),           # 9: 3H/2 x 6
            mp(3, 2, 2),                                             # 10
            cfgs._conv(18, 1, bn=False, act="linear"),               # 11
            cfgs._yolo("0,1,2", cfgs.TINY_ANCHORS, 6, classes=1)]    # 12


def edge_shapes_region(width=26, height=22):
    """Max-pools with padding=0 on even and odd sizes, reorgs of odd and non-square sizes at stride 2 and 3, and a [region]
    head."""
    return [cfgs._net(width, height),
            cfgs._conv(8, 3),                                                    # 0: 22 x 26
            ("maxpool", {"size": "2", "stride": "2", "padding": "0"}),           # 1: 11 x 13
            ("reorg", {"stride": "2"}),                                          # 2: 5 x 6 x 32
            ("route", {"layers": "-2"}),                                         # 3: 11 x 13 x 8
            ("maxpool", {"size": "2", "stride": "2", "padding": "0"}),           # 4: 5 x 6
            ("route", {"layers": "-1, -3"}),                                     # 5: 5 x 6 x 40
            ("route", {"layers": "0"}),                                          # 6: 22 x 26 x 8
            ("reorg", {"stride": "3"}),                                          # 7: 7 x 8 x 72
            ("maxpool", {"size": "5", "stride": "1"}),                           # 8: 7 x 8
            cfgs._conv(40, 1, bn=False, act="linear"),                           # 9
            cfgs._region("1.08,1.19,  3.42,4.41,  6.63,11.38,  9.42,5.11,  16.62,10.52", 3)]   # 10


# name -> (section builder, input size, weight seed, image seed)
ZOO = {
    "tiny64": (lambda: cfgs.slim(cfgs.yolov3_tiny, 2, 64, 64), 64, 11, 101),
    "xnor64": (lambda: cfgs.slim(cfgs.tiny_yolo_obj_xnor, 2, 64, 64), 64, 12, 102),
    "v3_32": (lambda: cfgs.slim(cfgs.yolov3, 4, 32, 32), 32, 13, 103),
    "spp32": (lambda: cfgs.slim(cfgs.yolov3_spp, 4, 32, 32), 32, 14, 104),
    "v2voc32": (lambda: cfgs.slim(cfgs.yolov2_voc, 4, 32, 32), 32, 15, 105),
    # non-square inputs (H != W): name -> builder uses (width, height)
    "tiny_w96_h64": (lambda: cfgs.slim(cfgs.yolov3_tiny, 2, 96, 64), (64, 96), 17, 107),
    "v3_w64_h96": (lambda: cfgs.slim(cfgs.yolov3, 4, 64, 96), (96, 64), 18, 108),
    "tinyvoc64": (lambda: cfgs.slim(cfgs.tiny_yolo_voc, 2, 64, 64), 64, 16, 106),
    "edges_yolo_w40_h24": (edge_shapes_yolo, (24, 40), 19, 109),
    "edges_region_w26_h22": (edge_shapes_region, (22, 26), 20, 110),
}


_WRITTEN = {}    # cfg path -> (sections, seed) it was written with in this session


def write_net(workdir, name, secs, seed, weights=None):
    """workdir/name.cfg and .weights for the sections `secs`, written once per session: the weights of cfgs.write_weights
    at `seed`, or what weights(path) writes, `seed` then naming that content.  A name written earlier with the same sections
    and seed is reused as it is (the 608 x 608 weights take a while to write); with other ones it is an error, so no test
    reads another test's network by accident."""
    cfg = os.path.join(workdir, name + ".cfg")
    wts = os.path.join(workdir, name + ".weights")
    key = (repr(secs), seed)
    if cfg in _WRITTEN:
        assert _WRITTEN[cfg] == key, f"{cfg} was written earlier in this session with other sections or another seed"
        return cfg, wts
    cfgs.write_cfg(secs, cfg)
    if weights is None:
        cfgs.write_weights(secs, wts, seed=seed)
    else:
        weights(wts)
    _WRITTEN[cfg] = key
    return cfg, wts


def model_files(name, workdir):
    build, size, wseed, _ = ZOO[name]
    return write_net(workdir, name, build(), wseed)


def images(name, batch):
    _, size, _, iseed = ZOO[name]
    h, w = size if isinstance(size, tuple) else (size, size)
    return cfgs.synthetic_images(batch, 3, h, w, seed=iseed)


def have_ref():
    from oracle import ref
    return ref.available("scalar")


def rel_l2(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def bits_equal(a, b):
    a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def ulp_diff(a, b, bf16):
    """distance in f32 (or, for bf16 values, bf16) units in the last place"""
    def key(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    d = np.abs(key(a) - key(b))
    return d >> 16 if bf16 else d


def bf16_round(a):
    """round-to-nearest-even float32 -> bfloat16 -> float32"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return (r & 0xFFFFFFFF).astype(np.uint32).view(np.float32).reshape(np.shape(a))


def logistic_bound(v):
    """|__fdividef(1, 1 + __expf(-v)) - 1 / (1 + exp(-v))| bound (CUDA C Programming Guide, intrinsic functions): __expf(x)
    is within 2 + floor(|1.173 x|) ulp, __fdividef within 2 ulp for a divisor in [2^-126, 2^126]; the 1 + e add rounds
    once more (1/2 ulp).  The relative error of 1 + e is at most that of e, so the result is within
    (2 + floor(|1.173 v|) + 0.5 + 2) ulp of an f32 value, relative to the result."""
    return (4.5 + np.floor(np.abs(1.173 * v))) * 2.0 ** -23


# ---- engine networks ----------------------------------------------------------------------------------------------------
def load(cfg, wts, batch, quantized=0, precision=None, fuse=None, keep_counts=False):
    """yb.load_network, then the precision, the `fuse` option and raw-count keeping where given"""
    import yolo2_light_b200 as yb
    net = yb.load_network(cfg, wts, batch=batch, quantized=quantized)
    if precision is not None:
        net.set_precision(precision)
    if fuse is not None:
        net.set_option("fuse", int(fuse))
    if keep_counts:
        net.set_option("keep_counts", 1)
    return net


def fetched(net, i, quantized=False):
    """layer i's output, or None where the engine does not materialise it (fused into another op)"""
    import yolo2_light_b200 as yb
    try:
        return net.fetch_layer(i, quantized=quantized)
    except yb.YbError:
        return None


def fetch_all(net, quantized=False):
    """every layer output the engine materialises, by index"""
    got = {i: fetched(net, i, quantized) for i in range(net.n)}
    return {i: o for i, o in got.items() if o is not None}


def profile_kinds(net, quantized=False):
    """layer -> the kinds of the ops Network.profile ran for it"""
    kinds = {}
    for li, kind, _ in net.profile(quantized=quantized):
        kinds.setdefault(li, []).append(kind)
    return kinds


# ---- the oracle ---------------------------------------------------------------------------------------------------------
def oracle_layer(L, i, x, rule, frm=None, xnor_rule=0):
    """Layer i (layer dict L) of the oracle on its input x (frm: a shortcut's `from` output), under the integer rule of
    `quantized` = rule (0 none, 1 the CPU rule, 2 the GPU rule) and the XNOR rule (rule_oracle.conv_arith).  Returns (output,
    the raw XNOR results or INT8 accumulators, or None)."""
    from oracle import port
    import rule_oracle
    t = L["type_name"]
    if t == "MAXPOOL":
        return port.maxpool(x, L["size"], L["stride"], L["pad"]), None
    if t == "UPSAMPLE":
        return port.upsample(x, L["stride"], L["scale"]), None
    if t == "REORG":
        return port.reorg(x, L["stride"]), None
    if t == "SHORTCUT":
        return port.shortcut(x, frm, L["activation"]), None
    assert t == "CONVOLUTIONAL", t
    layers = [None] * i + [L]    # conv_arith looks at layer i and the one behind it, which a lone layer does not have
    return rule_oracle.conv(L, rule_oracle.conv_arith(layers, i, rule, xnor_rule), x, want_raw=True)


def oracle_outs(net, x, rule, xnor_rule=0):
    """every layer's output of the oracle (rule_oracle.forward), image by image, concatenated over the batch"""
    import rule_oracle
    per_image = [rule_oracle.forward(net.layers, x[b:b + 1], rule, xnor_rule) for b in range(x.shape[0])]
    return [np.concatenate([pi[i] for pi in per_image], axis=0) for i in range(net.n)]


def xnor_gpu_layers(layers, quantized=0):
    """convolution -> its arithmetic under the GPU XNOR rule, for the XNOR layers that run as XNOR (not as INT8 under the
    GPU INT8 rule, quantized = 2); raises rule_oracle.Rejected where the engine refuses the network"""
    import rule_oracle
    ar = {i: rule_oracle.conv_arith(layers, i, quantized, rule_oracle.XNOR_GPU)
          for i, L in enumerate(layers) if L["type_name"] == "CONVOLUTIONAL"}
    return {i: a for i, a in ar.items() if a in ("xnor_gpu", "pm1z_gpu")}


# ---- kernel names -------------------------------------------------------------------------------------------------------
SIDES = {2: "SIDE_S8", 3: "SIDE_PM1_S8", 4: "SIDE_BITS"}      # yb::SideFmt values

_MANGLED_ARGS = [
    (re.compile(r"Li(\d+)E"), lambda m: m[1]),
    (re.compile(r"Lb([01])E"), lambda m: "true" if m[1] == "1" else "false"),
    (re.compile(r"LN(?:S_|2yb)7SideFmtE(\d+)E"), lambda m: SIDES[int(m[1])]),
    (re.compile(r"13__nv_bfloat16"), lambda m: "bf16"),
    (re.compile(r"f"), lambda m: "float"),
]
_POLICY = re.compile(r"N(?:S_|2yb)(\d+)")


def _demangled_arg(a):
    a = a.strip()
    m = re.fullmatch(r"\((?:yb::)?SideFmt\)(\d+)", a)
    if m:
        return SIDES[int(m[1])]
    if a == "__nv_bfloat16":
        return "bf16"
    return re.sub(r"<.*", "", a.replace("yb::", "")).strip()     # a policy: its name only


def kernel_inst(name):
    """(kernel, template arguments) of a kernel name as cudaFuncGetName gives it: mangled, or demangled.  A policy type
    argument (k_conv_simt's) is given by its name alone."""
    if name.startswith("_Z"):
        m = re.match(r"_ZN2ybL?(\d+)", name)
        assert m, name
        pos = m.end() + int(m[1])
        base, args = name[m.end():pos], []
        if name.startswith("I", pos):
            pos += 1
            while name[pos] != "E":
                p = _POLICY.match(name, pos)
                if p:
                    args.append(name[p.end():p.end() + int(p[1])])
                    break
                for rx, val in _MANGLED_ARGS:
                    a = rx.match(name, pos)
                    if a:
                        args.append(val(a))
                        pos = a.end()
                        break
                else:
                    raise ValueError(f"template argument at {pos} of {name}")
        return base, tuple(args)
    m = re.search(r"(k_\w+)(<?)", name)
    assert m, name
    base, args = m[1], []
    if m[2]:
        depth, cur = 1, ""
        for ch in name[m.end():]:
            depth += (ch == "<") - (ch == ">")
            if depth == 0 or (depth == 1 and ch == ","):
                args.append(_demangled_arg(cur))
                cur = ""
                if depth == 0:
                    break
            else:
                cur += ch
    return base, tuple(args)


def kernel_is(name, base):
    """name (mangled or not) is kernel `base`, not a longer kernel name that starts with it"""
    return name is not None and kernel_inst(name)[0] == base


# ---- networks and frames that several test files run ---------------------------------------------------------------------
def tcnet(size=64):
    """Exercises every tile configuration of k_conv_tc: BK 16/32/64, BN 32/64/128/256, 3x3 s1, 3x3 s2, 1x1, fused
    shortcut, concat slice output, f32 head with 255 filters."""
    c = cfgs._conv
    s = [cfgs._net(size, size),
         c(16, 3),                   # 0 stem (CUDA cores, C=3)
         c(32, 3, 2),                # 1 s2, BK16, BN32
         c(64, 3),                   # 2 s1, BK32, BN64
         c(32, 1),                   # 3 1x1, BK64, BN32
         c(64, 3),                   # 4 3x3 + fused shortcut
         ("shortcut", {"from": "-3", "activation": "linear"}),   # 5
         c(128, 3, 2),               # 6 s2, BK64, BN128
         c(64, 1),                   # 7
         c(128, 3),                  # 8
         ("shortcut", {"from": "-3", "activation": "linear"}),   # 9
         c(256, 3, 2),               # 10 s2 BN256
         c(128, 1),                  # 11
         c(256, 3),                  # 12
         c(320, 1),                  # 13 two filter tiles (256 + 64)
         c(255, 1, bn=False, act="linear"),   # 14 head, f32 out, n=255
         cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9),              # 15
         ("route", {"layers": "-4"}),                            # 16 -> layer 12
         c(64, 1),                   # 17
         ("upsample", {"stride": "2"}),                          # 18 writes a concat slice
         ("route", {"layers": "-1, 9"}),                         # 19 concat(64 + 128) = 192 channels
         c(128, 3),                  # 20 reads the concat (C=192, BK64)
         c(255, 1, bn=False, act="linear"),   # 21
         cfgs._yolo("3,4,5", cfgs.COCO_ANCHORS, 9)]              # 22
    return s


def s2chain():
    c = cfgs._conv
    return [cfgs._net(64, 64),
            c(32, 3),                   # 0 stem
            c(64, 3, 2),                # 1 s2, C=32
            c(64, 3),                   # 2 s1 over layer 1's borders
            c(128, 3, 2),               # 3 s2
            c(128, 3),                  # 4
            c(256, 3, 2),               # 5 s2, up to 256 filters per tile
            c(256, 3),                  # 6
            c(255, 1, bn=False, act="linear"),
            cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9)]


def widenet():
    """Fused shortcuts on 256-filter layers, a 1x1 and a 3x3, and a masked second filter tile."""
    c = cfgs._conv
    return [cfgs._net(32, 32),
            c(32, 3),
            c(64, 3, 2),
            c(256, 1),                  # 2
            c(128, 1),                  # 3
            c(256, 3),                  # 4 + fused shortcut
            ("shortcut", {"from": "-3", "activation": "linear"}),   # 5
            c(256, 1),                  # 6 + fused shortcut (1x1)
            ("shortcut", {"from": "-2", "activation": "linear"}),   # 7
            c(320, 3),                  # 8
            c(255, 1, bn=False, act="linear"),
            cfgs._yolo("0,1,2", cfgs.COCO_ANCHORS, 9)]


def bigger(name, workdir, w, h):
    """The slim zoo nets on a larger input: more grid cells -> a few hundred candidates per image."""
    build = {"tiny": cfgs.yolov3_tiny, "v3": cfgs.yolov3, "xnor": cfgs.tiny_yolo_obj_xnor, "v2voc": cfgs.yolov2_voc}[name]
    secs = cfgs.slim(build, 4 if name in ("v3", "v2voc") else 2, w, h)
    return write_net(workdir, f"det_{name}_{w}x{h}", secs, 41)


def sorted_rows(rows):
    """detection rows in the order of their boxes"""
    if rows.shape[0] == 0:
        return rows
    return rows[np.lexsort(rows[:, :4].T[::-1])]


def frames(sizes, seed):
    """random u8 HWC frames of the (w, h) sizes"""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for w, h in sizes]


# (w, h): 1 pixel wide, 1 pixel high, the network size (64), upscales, a >= 3x downscale, odd sizes, and a frame whose rows
# are wider than the resize kernel stages in shared memory
INPUT_SETS = [[(1, 40), (50, 1), (64, 64), (33, 17)],
              [(200, 197), (97, 131), (4500, 5)],
              [(7, 9)]]


def mixed_net(kind, workdir):
    """A batch-3 network for the mixed-frame tests and whether it runs quantized: the 8-bit-stem s2chain in bf16, or tiny64
    / xnor64 of the zoo in the precision the kind names."""
    import yolo2_light_b200 as yb
    if kind == "s2chain":
        cfg, wts = write_net(workdir, "frames_s2chain64", s2chain(), 61)
        return load(cfg, wts, 3, precision=yb.YB_PREC_BF16_TC), False
    name, q, prec = {"tiny64_fp32": ("tiny64", 0, yb.YB_PREC_FP32), "tiny64_bf16": ("tiny64", 0, yb.YB_PREC_BF16_TC),
                     "tiny64_q1": ("tiny64", 1, yb.YB_PREC_BF16_TC), "xnor64": ("xnor64", 0, yb.YB_PREC_BF16_TC)}[kind]
    cfg, wts = model_files(name, workdir)
    return load(cfg, wts, 3, quantized=q, precision=prec), bool(q)


# ---- the mAP data set -----------------------------------------------------------------------------------------------------
def write_bmp(path, img):   # img: u8 [h, w, 3] RGB
    h, w, _ = img.shape
    row = (3 * w + 3) // 4 * 4
    data = bytearray()
    for y in range(h - 1, -1, -1):
        line = img[y, :, ::-1].tobytes()
        data += line + b"\0" * (row - len(line))
    hdr = b"BM" + (54 + len(data)).to_bytes(4, "little") + b"\0\0\0\0" + (54).to_bytes(4, "little")
    dib = (40).to_bytes(4, "little") + w.to_bytes(4, "little") + h.to_bytes(4, "little") + (1).to_bytes(2, "little") + \
        (24).to_bytes(2, "little") + (0).to_bytes(4, "little") + len(data).to_bytes(4, "little") + \
        (2835).to_bytes(4, "little") * 2 + (0).to_bytes(4, "little") * 2
    open(path, "wb").write(hdr + dib + bytes(data))


def check_map_accounting(name, iou_thresh, workdir):
    """Writes the data set workdir/mapset_<name>_<iou %> (BMP images, labels, the reference's validate_detector_map output in
    ref_stdout.txt) and checks yb_map_evaluate's accounting against that output."""
    import yolo2_light_b200 as yb
    from oracle import ref
    cfg, wts = model_files(name, workdir)
    rnet = ref.RefNet(cfg, wts, 1, 0, 7)
    classes = rnet.layers[-1]["classes"]
    root = os.path.join(workdir, f"mapset_{name}_{int(iou_thresh * 100)}")
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    os.makedirs(os.path.join(root, "labels"), exist_ok=True)
    rng = np.random.default_rng(11)
    nimg = 7
    rows, truth, paths = [], [], []
    for k in range(nimg):
        img = rng.integers(0, 256, size=(72 + 4 * k, 80, 3), dtype=np.uint8)
        path = os.path.join(root, "images", f"img{k}.bmp")
        write_bmp(path, img)
        paths.append(path)
        x = ref.load_resize_u8(img, rnet.width, rnet.height)[None]      # what load_image + resize_image hand to the net
        rnet.predict(x)
        r = np.delete(rnet.get_boxes(1, 1, 0.005, 0.45), 5, axis=1)      # get_network_boxes(net, 1, 1, .005, ...) + NMS
        rows.append(r)
        # labels: some of the strongest detections (true positives), jittered copies (IoU near the threshold), strays
        lab = []
        if r.shape[0]:
            best = np.argsort(-r[:, 5:].max(axis=1))[:4]
            for j, i in enumerate(best):
                cls = int(np.argmax(r[i, 5:]))
                box = r[i, :4].astype(np.float64)
                if j % 2:
                    box = box * (1.0 + 0.08 * rng.standard_normal(4))
                lab.append((cls, *[round(float(v), 4) for v in box]))
        lab.append((int(rng.integers(0, classes)), 0.5, 0.5, 0.2, 0.3))
        if k == 3:
            lab = []                                                     # an image without labels (no file at all)
        else:
            with open(os.path.join(root, "labels", f"img{k}.txt"), "w") as f:
                for cls, bx, by, bw, bh in lab:
                    f.write(f"{cls} {bx:.4f} {by:.4f} {bw:.4f} {bh:.4f}\n")
        for cls, bx, by, bw, bh in lab:
            truth.append((k, cls, float(f"{bx:.4f}"), float(f"{by:.4f}"), float(f"{bw:.4f}"), float(f"{bh:.4f}")))
    open(os.path.join(root, "valid.txt"), "w").write("\n".join(paths) + "\n")
    open(os.path.join(root, "names.txt"), "w").write("\n".join(f"c{i}" for i in range(classes)) + "\n")
    datacfg = os.path.join(root, "data.cfg")
    open(datacfg, "w").write(f"classes = {classes}\nvalid = {root}/valid.txt\nnames = {root}/names.txt\n")

    out = ref.validate_map(datacfg, cfg, wts, 0.24, 0, iou_thresh, os.path.join(root, "ref_stdout.txt"))
    ap_ref = {int(m.group(1)): float(m.group(2)) for m in re.finditer(r"class_id = (\d+), name = \S+,\s+ap = ([0-9.]+) %", out)}
    m = re.search(r"(?:mean average precision \(mAP\)|average precision \(AP\)) = ([0-9.]+)", out)
    assert m and len(ap_ref) == classes, out[-400:]
    map_ref = float(m.group(1))
    tp, fp, fn, aiou = re.search(r"TP = (\d+), FP = (\d+), FN = (\d+), average IoU = ([0-9.]+) %", out).groups()
    prf = re.search(r"precision = ([0-9.]+), recall = ([0-9.]+), F1-score = ([0-9.]+)", out).groups()
    ndet = int(re.search(r"detections_count = (\d+), unique_truth_count = (\d+)", out).group(1))

    mAP, ap, st = yb.api.map_evaluate(rows, np.array(truth, np.float32).reshape(-1, 6), classes, iou_thresh, 0.24)
    assert int(st["detections"]) == ndet
    assert (int(st["tp"]), int(st["fp"]), int(st["fn"])) == (int(tp), int(fp), int(fn))
    assert abs(mAP - map_ref) < 5e-7, (mAP, map_ref)                      # the reference prints %f
    for c in range(classes):
        assert abs(ap[c] * 100 - ap_ref[c]) <= 0.00501, (c, ap[c], ap_ref[c])   # printed with %2.2f
    assert abs(st["avg_iou"] * 100 - float(aiou)) <= 0.00501
    for mine, theirs in zip((st["precision"], st["recall"], st["f1"]), prf):
        assert abs(mine - float(theirs)) <= 0.00501 or (np.isnan(mine) and "nan" in theirs)
    assert int(tp) > 0 and mAP > 0                                       # the dataset exercises the matching at all
