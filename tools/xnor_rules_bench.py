"""Forward time of the two XNOR rules on tiny-yolo-obj_xnor 416 x 416: YB_XNOR_CPU (the reference CPU build's XNOR arithmetic)
and YB_XNOR_GPU (its GPU build's: the bit GEMM's FMA epilogue, zero-padded +-1 layers below 32 channels), at the default
precision, quantized = 0.

Synthetic seeded weights, batch --batch.  One network per rule (setting the rule drops a network's engines); the rules are
timed alternated, --rounds rounds each: per round and rule, CUDA events around --steps device-resident forwards after --warmup.
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

RULES = (("cpu", yb.YB_XNOR_CPU), ("gpu", yb.YB_XNOR_GPU))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    vals = [v.strip() for v in out.splitlines()[0].split(",")] if out.strip() else []
    return dict(zip(q.split(","), vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("xnor_rules_bench: no CUDA device")
    wd = tempfile.mkdtemp()
    stream = torch.cuda.Stream()   # a real (non-default) stream: the engine enqueues its forward on the caller's stream
    torch.cuda.set_stream(stream)
    result = {"card_before": card(), "net": "tiny-yolo-obj_xnor-416", "batch": a.batch, "steps": a.steps, "warmup": a.warmup}
    secs = cfgs.tiny_yolo_obj_xnor(416, 416)
    cfg = cfgs.write_cfg(secs, os.path.join(wd, "xnor.cfg"))
    wts = cfgs.write_weights(secs, os.path.join(wd, "xnor.weights"), seed=3)
    x = torch.from_numpy(cfgs.synthetic_images(a.batch, 3, 416, 416, seed=4)).cuda()
    nets = {}
    for name, rule in RULES:
        nets[name] = yb.load_network(cfg, wts, batch=a.batch)
        nets[name].set_xnor_rule(rule)
        for _ in range(a.warmup):   # build every engine and warm it up before any timing
            nets[name].forward_device(x.data_ptr(), stream=stream.cuda_stream)
    torch.cuda.synchronize()
    times = {name: [] for name, _ in RULES}
    for _ in range(a.rounds):
        for name, _ in RULES:
            net = nets[name]
            for _ in range(a.warmup):
                net.forward_device(x.data_ptr(), stream=stream.cuda_stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.steps):
                net.forward_device(x.data_ptr(), stream=stream.cuda_stream)
            e1.record(stream)
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    result["ms_per_batch"] = {k: [round(t, 4) for t in v] for k, v in times.items()}
    result["ms_per_batch_median"] = {k: round(float(np.median(v)), 4) for k, v in times.items()}
    result["img_per_s_median"] = {k: round(a.batch * 1000.0 / float(np.median(v)), 1) for k, v in times.items()}
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
