"""Serving throughput with and without drawing the detections into the device frames (yb_network_submit_device_frames vs
yb_network_submit_device_frames_draw).

Workload: yolov3 at 608x608, batch 16, bf16 tensor cores, synthetic weights; 1920x1080 NV12 frames in device memory, three
tickets in flight.  Batch i reads frame set i % 3 and is ordered with caller stream i % 3, as a decoder with three surface
pools would hand them over: the drawing call makes its stream wait for the draw, so the next write into a set (here: the
next read of it) comes after the draw, and the other sets go on meanwhile.  The two calls are alternated for --rounds
rounds in one process.  Also reported: the device time per batch of k_det_select and k_det_draw<NV12> (torch.profiler CUDA
activity, a pass of its own), the boxes drawn per image, and the card's name and power limit, read in the same run.  The
synthetic weights get raised class biases in the three detection heads (raise_class_biases), so that boxes are drawn.

  python tools/draw_bench.py [--batches 30] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import yolo2_light_b200 as yb  # noqa: E402
from yolo2_light_b200 import cfgs  # noqa: E402
from frames_bench import card, run_pipeline  # noqa: E402

W, H = 1920, 1080
NET, BATCH, SETS = 608, 16, 3


def raise_class_biases(secs, path, by=6.0):
    """Adds `by` to the bias of every class channel of the convolutions that feed the [yolo] layers, in the .weights file
    cfgs.write_weights wrote: untrained heads sit at objectness and class scores ~0.5, so prob = objectness * class score
    never passes a threshold that objectness passes, and nothing would be drawn.  With the class scores near 1 every
    candidate past the NMS is drawn."""
    shapes = cfgs.conv_shapes(secs)
    kinds = [s[0] for s in secs[1:]]
    convs = [L for L in shapes if L["type"] in ("convolutional", "conv")]
    feeds = set()
    ci = -1
    for i, k in enumerate(kinds):
        if k in ("convolutional", "conv"):
            ci += 1
        elif k == "yolo":
            feeds.add(ci)
    buf = bytearray(open(path, "rb").read())
    off = 20
    for j, L in enumerate(convs):
        n, c, k = L["n"], L["c"], L["size"]
        if j in feeds:
            b = np.frombuffer(buf, "<f4", n, off).copy()
            for a in range(n // 85):
                b[a * 85 + 5:(a + 1) * 85] += by
            buf[off:off + 4 * n] = b.tobytes()
        off += 4 * n * (4 if L["bn"] else 1) + 4 * n * c * k * k
    assert off == len(buf), (off, len(buf))
    open(path, "wb").write(bytes(buf))


def kernel_us(submit, collect, batches, names):
    """Mean device time per launch of each kernel whose name contains one of `names`, in a profiled pass of its own."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_pipeline(submit, collect, batches)
        torch.cuda.synchronize()
    out = {}
    for n in names:
        ks = [e for e in prof.events() if n in e.name]
        us = [e.device_time if hasattr(e, "device_time") else e.cuda_time for e in ks]
        out[n] = (round(float(np.mean(us)), 1) if us else None, len(us))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=30, help="batches per timed pass (a multiple of 3)")
    ap.add_argument("--rounds", type=int, default=3, help="rounds of the two calls, alternated")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    wd = tempfile.mkdtemp(prefix="yb_draw_")
    secs = cfgs.MODELS["yolov3"](NET, NET)
    cfg, wts = os.path.join(wd, "m.cfg"), os.path.join(wd, "m.weights")
    cfgs.write_cfg(secs, cfg)
    cfgs.write_weights(secs, wts, seed=1)
    raise_class_biases(secs, wts)
    net = yb.load_network(cfg, wts, batch=BATCH)
    net.set_precision(yb.YB_PREC_BF16_TC)

    g = torch.Generator(device="cuda").manual_seed(7)
    sets = [list(torch.randint(0, 256, (BATCH, H * 3 // 2, W), dtype=torch.uint8, device="cuda", generator=g))
            for _ in range(SETS)]
    streams = [torch.cuda.Stream() for _ in range(SETS)]
    torch.cuda.synchronize()
    batches = [(sets[i % SETS], streams[i % SETS].cuda_stream) for i in range(a.batches)]

    # detection threshold as in frames_bench: untrained heads sit at objectness ~0.5; raise it until an image yields at most
    # a few hundred candidates
    thresh, cap = 0.5, 4096
    while thresh < 0.95:
        t = net.submit_device_frames(sets[0], thresh, fmt="nv12", max_rows=cap)
        _, cnt, _ = net.collect_detections(t)
        if int(cnt.max()) <= 300:
            break
        thresh = round(thresh + 0.01, 2)

    def collect(t):
        net.collect_detections(t, copy=False)

    def sub_plain(b):
        return net.submit_device_frames(b[0], thresh, fmt="nv12", max_rows=cap, stream=b[1])

    def sub_draw(b):
        return net.submit_device_frames_draw(b[0], thresh, fmt="nv12", max_rows=cap, stream=b[1])

    # drawing changes no detection, and how many boxes it draws
    d0, c0, _ = net.collect_detections(sub_plain(batches[0]))
    t = sub_draw(batches[0])
    d1, c1, _ = net.collect_detections(t)
    same = bool(np.array_equal(c0, c1)) and all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(d0, d1))
    drawn = [len(s) for s in net.selected_detections(t)]

    for sub in (sub_plain, sub_draw):   # warm-up
        run_pipeline(sub, collect, batches[:6])
    times = {"plain": [], "draw": []}
    for _ in range(a.rounds):
        times["plain"].append(run_pipeline(sub_plain, collect, batches))
        times["draw"].append(run_pipeline(sub_draw, collect, batches))
    torch.cuda.synchronize()
    prof = kernel_us(sub_draw, collect, batches[:12], ["k_det_select", "k_det_draw", "k_det_nms"])

    nimg = a.batches * BATCH
    res = {
        "workload": f"yolov3-{NET} b{BATCH} bf16, {W}x{H} NV12 device frames, three tickets in flight",
        "card": card(),
        "images_per_pass": nimg,
        "det_thresh": thresh,
        "same_detections": same,
        "boxes_drawn_per_image": [min(drawn), round(float(np.mean(drawn)), 1), max(drawn)],
        "submit_device_frames_img_s": [round(nimg / x, 1) for x in times["plain"]],
        "submit_device_frames_draw_img_s": [round(nimg / x, 1) for x in times["draw"]],
        "k_det_select_us_per_batch": prof["k_det_select"][0],
        "k_det_draw_us_per_batch": prof["k_det_draw"][0],
        "k_det_nms_us_per_launch": prof["k_det_nms"][0],
        "launches_profiled": {k: v[1] for k, v in prof.items()},
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
