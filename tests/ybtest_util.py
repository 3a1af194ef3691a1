"""Shared helpers for the test-suite: small model zoo (generated cfg + seeded weights), reference/oracle access."""
import os
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


def model_files(name, workdir):
    build, size, wseed, _ = ZOO[name]
    secs = build()
    cfg = os.path.join(workdir, name + ".cfg")
    wts = os.path.join(workdir, name + ".weights")
    if not os.path.exists(cfg):
        cfgs.write_cfg(secs, cfg)
        cfgs.write_weights(secs, wts, seed=wseed)
    return cfg, wts


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
