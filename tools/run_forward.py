"""Runs N eager forwards of a workload (YB_NO_GRAPH=1 makes every kernel a plain launch) -- target for ncu."""
import argparse, os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import yolo2_light_b200 as yb
from yolo2_light_b200 import cfgs

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="yolov3"); ap.add_argument("--size", type=int, default=608)
ap.add_argument("--batch", type=int, default=16); ap.add_argument("--quantized", type=int, default=0)
ap.add_argument("--reps", type=int, default=1); ap.add_argument("--list", action="store_true")
ap.add_argument("--precision", choices=["bf16", "fp32"], default="bf16", help="fp32: YB_PREC_FP32, the exact f32 path")
a = ap.parse_args()
wd = tempfile.mkdtemp()
secs = cfgs.MODELS[a.model](a.size, a.size)
cfg = cfgs.write_cfg(secs, os.path.join(wd, "m.cfg")); wts = cfgs.write_weights(secs, os.path.join(wd, "m.weights"), seed=1)
net = yb.load_network(cfg, wts, batch=a.batch, quantized=a.quantized)
net.set_precision(yb.YB_PREC_FP32 if a.precision == "fp32" else yb.YB_PREC_BF16_TC)
x = cfgs.synthetic_images(a.batch, 3, a.size, a.size)
if a.list:
    net.predict(x, quantized=bool(a.quantized))
    for k, (li, kind, ms) in enumerate(net.profile(quantized=bool(a.quantized))):
        print(k, li, kind, f"{ms:.4f}")
else:
    for _ in range(a.reps):
        net.predict(x, quantized=bool(a.quantized))
