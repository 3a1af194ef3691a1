"""Serving throughput for frames that are already in device memory (yb_network_submit_device_frames).

Workload: yolov3 at 608x608, batch 16, bf16 tensor cores, synthetic weights; a stream of 1920x1080 frames, three tickets in
flight.  The same picture content goes in three ways:

  (a) NV12 frames in device memory (what a hardware video decoder writes) through submit_device_frames;
  (b) the same content as packed RGB frames in device memory through submit_device_frames;
  (c) the same RGB frames from pinned host memory through submit_frames_u8 (copied to the device with every batch).

The three are alternated for --rounds rounds in one process.  Also reported: k_resize_frames' device time per batch for
NV12 and for RGB device frames (torch.profiler CUDA activity, a pass of its own per format), the bytes the algorithm moves
(frames read + 12 * 608 * 608 per image written) and that over 3.35 TB/s (the H100 SXM's HBM3 data sheet figure) as the
time floor, and the card's name and power limit, read in the same run.

  python tools/device_frames_bench.py [--batches 30] [--rounds 3] [--out result.json]
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
from frames_bench import HBM_BPS, card, run_pipeline  # noqa: E402

W, H = 1920, 1080
NET, BATCH = 608, 16
POOL = 2 * BATCH        # distinct frames, cycled by the stream


def nv12_to_rgb(nv12):
    """torch uint8 [n, 3h/2, w] NV12 -> [n, h, w, 3] RGB on the device: BT.601 limited range, OpenCV's fixed-point form
    (the conversion YB_FRAME_NV12 specifies)."""
    import torch
    h = nv12.shape[1] // 3 * 2
    y = nv12[:, :h].int()
    uv = nv12[:, h:].int().reshape(nv12.shape[0], h // 2, -1, 2)
    u = uv[..., 0].repeat_interleave(2, 1).repeat_interleave(2, 2) - 128
    v = uv[..., 1].repeat_interleave(2, 1).repeat_interleave(2, 2) - 128
    yy = torch.clamp(y - 16, min=0) * 1220542 + (1 << 19)
    rgb = torch.stack([yy + 1673527 * v, yy - 852492 * v - 409993 * u, yy + 2116026 * u], -1) >> 20
    return rgb.clamp(0, 255).to(torch.uint8)


def resize_us(submit, collect, batches, fmt_id):
    """Mean device time of k_resize_frames<fmt_id> per batch, in a profiled pass of its own."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_pipeline(submit, collect, batches)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if f"k_resize_frames<{fmt_id}>" in e.name]
    us = [e.device_time if hasattr(e, "device_time") else e.cuda_time for e in ks]
    return (float(np.mean(us)) if us else float("nan")), len(us)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=30, help="batches per timed pass")
    ap.add_argument("--rounds", type=int, default=3, help="rounds of (a), (b), (c), alternated")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    wd = tempfile.mkdtemp(prefix="yb_device_frames_")
    secs = cfgs.MODELS["yolov3"](NET, NET)
    cfg, wts = os.path.join(wd, "m.cfg"), os.path.join(wd, "m.weights")
    cfgs.write_cfg(secs, cfg)
    cfgs.write_weights(secs, wts, seed=1)
    net = yb.load_network(cfg, wts, batch=BATCH)
    net.set_precision(yb.YB_PREC_BF16_TC)

    g = torch.Generator(device="cuda").manual_seed(7)
    nv12 = torch.randint(0, 256, (POOL, H * 3 // 2, W), dtype=torch.uint8, device="cuda", generator=g)
    rgb = nv12_to_rgb(nv12)
    pinned = yb.PinnedBuffer(POOL * H * W * 3, dtype=np.uint8)
    host = pinned.array.reshape(POOL, H, W, 3)
    host[:] = rgb.cpu().numpy()
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream().cuda_stream

    def batch_list(frames):
        return [[frames[(i * BATCH + j) % POOL] for j in range(BATCH)] for i in range(a.batches)]

    b_nv12, b_rgb, b_host = batch_list(list(nv12)), batch_list(list(rgb)), batch_list(list(host))

    # detection threshold as in frames_bench: untrained heads sit at objectness ~0.5; raise it until an image yields at most
    # a few hundred candidates
    thresh, cap = 0.5, 4096
    net.predict_frames_u8(b_host[0])
    while thresh < 0.95:
        _, cnt = net.detect_frames([(W, H)] * BATCH, thresh, 0.45, max_rows=cap)
        if int(cnt.max()) <= 300:
            break
        thresh = round(thresh + 0.01, 2)

    def collect(t):
        net.collect_detections(t, copy=False)

    def sub_nv12(b):
        return net.submit_device_frames(b, thresh, fmt="nv12", max_rows=cap, stream=stream)

    def sub_rgb(b):
        return net.submit_device_frames(b, thresh, fmt="rgb", max_rows=cap, stream=stream)

    def sub_host(b):
        return net.submit_frames_u8(b, thresh, 0.45, max_rows=cap)

    # the three ways give the same detections
    same = True
    for b in range(2):
        res = []
        for sub, bl in ((sub_nv12, b_nv12), (sub_rgb, b_rgb), (sub_host, b_host)):
            d, c, _ = net.collect_detections(sub(bl[b]))
            res.append((d, c))
        same &= all(np.array_equal(res[0][1], r[1]) and all(np.array_equal(x.view(np.uint32), y.view(np.uint32))
                                                             for x, y in zip(res[0][0], r[0])) for r in res[1:])

    for sub, bl in ((sub_nv12, b_nv12), (sub_rgb, b_rgb), (sub_host, b_host)):   # warm-up
        run_pipeline(sub, collect, bl[:6])
    t = {"a": [], "b": [], "c": []}
    for _ in range(a.rounds):
        t["a"].append(run_pipeline(sub_nv12, collect, b_nv12))
        t["b"].append(run_pipeline(sub_rgb, collect, b_rgb))
        t["c"].append(run_pipeline(sub_host, collect, b_host))
    torch.cuda.synchronize()

    nimg = a.batches * BATCH
    us_nv12, n_nv12 = resize_us(sub_nv12, collect, b_nv12[:12], 3)
    us_rgb, n_rgb = resize_us(sub_rgb, collect, b_rgb[:12], 0)
    written = 12 * NET * NET * BATCH
    bytes_nv12, bytes_rgb = W * H * 3 // 2 * BATCH + written, W * H * 3 * BATCH + written
    res = {
        "workload": f"yolov3-{NET} b{BATCH} bf16, {W}x{H} frames, three tickets in flight",
        "card": card(),
        "images_per_pass": nimg,
        "det_thresh": thresh,
        "same_detections": bool(same),
        "a_device_nv12_img_s": [round(nimg / x, 1) for x in t["a"]],
        "b_device_rgb_img_s": [round(nimg / x, 1) for x in t["b"]],
        "c_pinned_host_rgb_img_s": [round(nimg / x, 1) for x in t["c"]],
        "resize_launches_profiled": [n_nv12, n_rgb],
        "resize_us_per_batch_nv12": round(us_nv12, 1),
        "resize_us_per_batch_rgb": round(us_rgb, 1),
        "resize_bytes_per_batch_nv12": bytes_nv12,
        "resize_bytes_per_batch_rgb": bytes_rgb,
        "resize_hbm_floor_us_nv12": round(bytes_nv12 / HBM_BPS * 1e6, 1),
        "resize_hbm_floor_us_rgb": round(bytes_rgb / HBM_BPS * 1e6, 1),
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
