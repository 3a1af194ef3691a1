"""Serving throughput for a stream of frames of different sizes (yb_network_submit_frames_u8).

Workload: yolov3 at 608x608, batch 16, bf16 tensor cores, synthetic weights; 8-bit frames in pinned host memory from a
stream that cycles 640x480 / 1280x720 / 1920x1080 (so every batch mixes three sizes), three tickets in flight.  Reports

  (a) img/s of submit_frames_u8 on the mixed stream;
  (b) img/s of the same frames regrouped by size and sent through submit_u8 -- the best the one-size call can do, and only
      when the caller reorders its frames;
  (c) k_resize_frames' device time per batch of the mixed stream (torch.profiler CUDA activity, its own pass), the bytes the
      algorithm moves (frames read + 12 * 608 * 608 per image written) and that over 3.35 TB/s (the H100 SXM's HBM3 data
      sheet figure) as the time floor;
  (d) the card's name and power limit, read in the same run.

With --letterbox it measures letterboxing instead (yb_network_set_letterbox): the same mixed stream through
submit_frames_u8 with letterboxing on (letter = 1) against off (letter = 0), alternated for three pairs, and
k_resize_frames' device time per mixed batch for each, in profiler passes of their own.

  python tools/frames_bench.py [--batches 30] [--letterbox] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import yolo2_light_b200 as yb  # noqa: E402
from yolo2_light_b200 import cfgs  # noqa: E402

SIZES = [(640, 480), (1280, 720), (1920, 1080)]
NET, BATCH, HBM_BPS = 608, 16, 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def run_pipeline(submit, collect, batches):
    inflight = []
    t0 = time.perf_counter()
    for b in batches:
        if len(inflight) == 3:
            collect(inflight.pop(0))
        inflight.append(submit(b))
    while inflight:
        collect(inflight.pop(0))
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=30, help="mixed batches per timed pass (a multiple of 3)")
    ap.add_argument("--letterbox", action="store_true", help="letterbox on against off instead of (a) - (c)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    nb = max(3, a.batches // 3 * 3)
    nimg = nb * BATCH
    wd = tempfile.mkdtemp(prefix="yb_frames_")
    secs = cfgs.MODELS["yolov3"](NET, NET)
    cfg, wts = os.path.join(wd, "m.cfg"), os.path.join(wd, "m.weights")
    cfgs.write_cfg(secs, cfg)
    cfgs.write_weights(secs, wts, seed=1)
    net = yb.load_network(cfg, wts, batch=BATCH)
    net.set_precision(yb.YB_PREC_BF16_TC)

    # frame k of the stream has size SIZES[k % 3]; per size, the stream's frames of that size lie back to back in one
    # pinned buffer, so the regrouped batches of (b) are stacked arrays
    per_size = nimg // 3
    rng = np.random.default_rng(7)
    pools = []
    for w, h in SIZES:
        pb = yb.PinnedBuffer(per_size * h * w * 3, dtype=np.uint8)
        pb.array[:] = rng.integers(0, 256, size=pb.array.size, dtype=np.uint8)
        pools.append((pb, pb.array.reshape(per_size, h, w, 3)))
    stream = [pools[k % 3][1][k // 3] for k in range(nimg)]
    mixed = [stream[i:i + BATCH] for i in range(0, nimg, BATCH)]
    grouped = [pools[s][1][i:i + BATCH] for i in range(0, per_size, BATCH) for s in range(3)]

    # detection threshold: untrained heads sit at objectness ~0.5; raise it until an image yields at most a few hundred
    # candidates, as a trained detector would hand to the NMS
    thresh, cap = 0.5, 4096
    net.predict_frames_u8(mixed[0])
    while thresh < 0.95:
        _, cnt = net.detect_frames([(f.shape[1], f.shape[0]) for f in mixed[0]], thresh, 0.45, max_rows=cap)
        if int(cnt.max()) <= 300:
            break
        thresh = round(thresh + 0.01, 2)

    def collect(t):
        net.collect_detections(t, copy=False)

    def sub_mixed(b):
        return net.submit_frames_u8(b, thresh, 0.45, max_rows=cap)

    def sub_grouped(b):
        return net.submit_u8(b, thresh, 0.45, max_rows=cap)

    if a.letterbox:
        res = letterbox_leg(net, mixed, thresh, cap, collect, nimg, nb)
        res["card"] = card()
        emit(res, a.out)
        return

    run_pipeline(sub_mixed, collect, mixed[:6])          # warm-up: engine, slots, buffers, both paths
    run_pipeline(sub_grouped, collect, grouped[:6])
    ta, tb = [], []
    for _ in range(3):                                   # alternate the two, three pairs
        ta.append(run_pipeline(sub_mixed, collect, mixed))
        tb.append(run_pipeline(sub_grouped, collect, grouped))

    # (c) resize kernel time: its own pass under the profiler
    dev_us = resize_times(sub_mixed, collect, mixed[:12])
    resize_us = float(np.mean(dev_us)) if dev_us else float("nan")
    bytes_per_batch = sum(f.size for b in mixed for f in b) / nb + 12 * NET * NET * BATCH
    floor_us = bytes_per_batch / HBM_BPS * 1e6

    res = {
        "workload": f"yolov3-{NET} b{BATCH} bf16, pinned 8-bit frames cycling "
                    + " / ".join(f"{w}x{h}" for w, h in SIZES) + ", three tickets in flight",
        "card": card(),
        "images_per_pass": nimg,
        "det_thresh": thresh,
        "a_submit_frames_u8_img_s": [round(nimg / t, 1) for t in ta],
        "b_regrouped_submit_u8_img_s": [round(nimg / t, 1) for t in tb],
        "c_resize_launches_profiled": len(dev_us),
        "c_resize_us_per_batch": round(resize_us, 1),
        "c_resize_bytes_per_batch": int(bytes_per_batch),
        "c_resize_hbm_floor_us": round(floor_us, 1),
        "c_resize_share_of_hbm_floor": round(floor_us / resize_us, 3) if dev_us else None,
    }
    emit(res, a.out)


def resize_times(submit, collect, batches):
    """k_resize_frames' device time (us) of each launch of one pipelined pass, under torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_pipeline(submit, collect, batches)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if "k_resize_frames" in e.name]
    return [e.device_time if hasattr(e, "device_time") else e.cuda_time for e in ks]


def letterbox_leg(net, mixed, thresh, cap, collect, nimg, nb):
    """The mixed stream letterboxed (letter = 1) against stretched (letter = 0), alternated; then k_resize_frames per batch
    for each in a profiler pass of its own."""
    def submitter(on):
        def sub(b):
            net.set_letterbox(on)
            return net.submit_frames_u8(b, thresh, 0.45, letter=int(on), max_rows=cap)
        return sub

    sub_on, sub_off = submitter(True), submitter(False)
    run_pipeline(sub_on, collect, mixed[:6])            # warm-up both
    run_pipeline(sub_off, collect, mixed[:6])
    t_on, t_off = [], []
    for _ in range(3):
        t_off.append(run_pipeline(sub_off, collect, mixed))
        t_on.append(run_pipeline(sub_on, collect, mixed))
    us_off = resize_times(sub_off, collect, mixed[:12])
    us_on = resize_times(sub_on, collect, mixed[:12])
    net.set_letterbox(False)
    return {
        "workload": f"yolov3-{NET} b{BATCH} bf16, pinned 8-bit frames cycling "
                    + " / ".join(f"{w}x{h}" for w, h in SIZES) + ", three tickets in flight, letterbox on vs off",
        "images_per_pass": nimg,
        "batches_per_pass": nb,
        "det_thresh": thresh,
        "stretched_submit_frames_u8_img_s": [round(nimg / t, 1) for t in t_off],
        "letterboxed_submit_frames_u8_img_s": [round(nimg / t, 1) for t in t_on],
        "resize_launches_profiled": [len(us_off), len(us_on)],
        "stretched_resize_us_per_batch": round(float(np.mean(us_off)), 1) if us_off else None,
        "letterboxed_resize_us_per_batch": round(float(np.mean(us_on)), 1) if us_on else None,
    }


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        open(out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
