"""Forward time of the three INT8 rules on one network: 0 (no INT8 layer), 1 (the CPU build's rule, yolov2_forward_network_q)
and 2 (the GPU build's rule, l.quantized with the saturating conversion and the unscaled epilogue), at the default precision.

yolov3-tiny 416 batch 64 and yolov3 608 batch 16, synthetic seeded weights, the cfg parsed with quantized = 1.  The rules are
timed alternated, three rounds each: per round and rule, CUDA events around --steps device-resident forwards after --warmup.
Prints one JSON line with the card's name, power limit and SM clocks read in the same call; --out also writes it to a file."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import yolo2_light_b200 as yb  # noqa: E402
from yolo2_light_b200 import cfgs  # noqa: E402

NETS = (("yolov3-tiny-416", lambda: cfgs.yolov3_tiny(416, 416), 416, 64),
        ("yolov3-608", lambda: cfgs.yolov3(608, 608), 608, 16))
RULES = (0, 1, 2)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    vals = [v.strip() for v in out.splitlines()[0].split(",")] if out.strip() else []
    return dict(zip(q.split(","), vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("int8_rules_bench: no CUDA device")
    wd = tempfile.mkdtemp()
    stream = torch.cuda.Stream()   # a real (non-default) stream: the engine enqueues its forward on the caller's stream
    torch.cuda.set_stream(stream)
    assert stream.cuda_stream != 0
    result = {"card_before": card(), "steps": a.steps, "warmup": a.warmup, "nets": {}}
    for name, build, size, B in NETS:
        secs = build()
        cfg = cfgs.write_cfg(secs, os.path.join(wd, name + ".cfg"))
        wts = cfgs.write_weights(secs, os.path.join(wd, name + ".weights"), seed=3)
        net = yb.load_network(cfg, wts, batch=B, quantized=1)
        x = torch.from_numpy(cfgs.synthetic_images(B, 3, size, size, seed=4)).cuda()
        for q in RULES:   # build every engine and warm it up before any timing
            for _ in range(a.warmup):
                net.forward_device(x.data_ptr(), quantized=q, stream=stream.cuda_stream)
        torch.cuda.synchronize()
        times = {q: [] for q in RULES}
        for _ in range(a.rounds):
            for q in RULES:
                for _ in range(a.warmup):
                    net.forward_device(x.data_ptr(), quantized=q, stream=stream.cuda_stream)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(a.steps):
                    net.forward_device(x.data_ptr(), quantized=q, stream=stream.cuda_stream)
                e1.record(stream)
                e1.synchronize()
                times[q].append(e0.elapsed_time(e1) / a.steps)
        result["nets"][name] = {
            "batch": B,
            "int8_layers": {str(q): sum(1 for i, l in enumerate(net.layers) if l["type_name"] == "CONVOLUTIONAL" and
                                        ((q == 1 and i >= 1 and l["activation"] != yb.api.YB_LINEAR) or (q == 2 and l["quantized"])))
                            for q in RULES},
            "ms_per_step": {str(q): [round(t, 4) for t in times[q]] for q in RULES},
            "ms_per_step_median": {str(q): round(float(np.median(times[q])), 4) for q in RULES},
            "img_per_s_median": {str(q): round(B * 1000.0 / float(np.median(times[q])), 1) for q in RULES},
        }
        del net
        torch.cuda.synchronize()
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
