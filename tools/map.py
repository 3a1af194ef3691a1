"""mAP of a network on a darknet-style validation set (SURVEY 8f row 4) -- what `darknet detector map data cfg weights`
does in the reference (validate_detector_map, additionally.c:4541-4898), with the forward, the image resize and the
decode + NMS on the GPU and the reference's bookkeeping (yb_map_evaluate) on the host.

  python tools/map.py obj.data net.cfg net.weights [--quantized] [--batch 16] [--iou 0.5] [--thresh 0.24]

Images: 24-bit BMP / binary PPM.  Every batch takes the next --batch images whatever their sizes, each resized and
decoded on its own terms (yb_network_predict_frames_u8 + yb_network_detect_frames); the last batch may be partial.
"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import yolo2_light_b200 as yb
from yolo2_light_b200 import dataset

ap = argparse.ArgumentParser()
ap.add_argument("data"); ap.add_argument("cfg"); ap.add_argument("weights")
ap.add_argument("--quantized", action="store_true"); ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--iou", type=float, default=0.5); ap.add_argument("--thresh", type=float, default=0.24)
ap.add_argument("--max-rows", type=int, default=8192)
a = ap.parse_args()
paths, names, truth = dataset.load_validation_set(a.data)
net = yb.load_network(a.cfg, a.weights, batch=a.batch, quantized=int(a.quantized))
classes = max(net.layer_desc(i).classes for i in range(net.n))
mAP, aps, st = dataset.evaluate_map(net, paths, truth, classes, a.iou, a.thresh, a.max_rows, a.quantized,
                                    progress=lambda i, n: print(f"\r{i}/{n}", end="", file=sys.stderr), mixed_sizes=True)
print(file=sys.stderr)
for c in range(classes):
    print(f"class_id = {c}, name = {names[c] if c < len(names) else c}, \t ap = {aps[c] * 100:2.2f} % ")
print(f" for thresh = {a.thresh:1.2f}, precision = {st['precision']:1.2f}, recall = {st['recall']:1.2f}, F1-score = {st['f1']:1.2f} ")
print(f" for thresh = {a.thresh:0.2f}, TP = {int(st['tp'])}, FP = {int(st['fp'])}, FN = {int(st['fn'])}, average IoU = {st['avg_iou'] * 100:2.2f} % ")
print(f"\n mean average precision (mAP) = {mAP:f}, or {mAP * 100:2.2f} % ")
