"""Records tests/golden/tc_plans.json: the tensor-core plan (Network.tc_plan) of every layer that has one, for every case of
make_engine_plans.cases() (every model of cfgs.MODELS, precision and fusion setting; 128 x 128, batch 2).  Needs a GPU:
    python tests/golden/make_tc_plans.py [OUT.json]

A plan's filter tile width and grid depend on the SM count, so the file names the card it was recorded on and its SM count;
tests/test_gpu_tc_plans.py rebuilds the same cases and compares on a card with the same SM count.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import make_engine_plans as plans  # noqa: E402
from yolo2_light_b200.api import TC_PLAN_FIELDS as FIELDS  # noqa: E402

# plan switches for experiments and tests: none of them may be set while recording or comparing
PLAN_ENV = ("YB_TC_BN", "YB_TC_GRID", "YB_TC_NO_BSTAT", "YB_NO_STEM_S2_FUSE")


def device():
    import torch
    prop = torch.cuda.get_device_properties(0)
    return prop.name, prop.multi_processor_count


def record(net, prec, fuse, no_s2):
    """Builds the engine of one case (make_engine_plans.record) and returns {layer: plan} of its tensor-core layers, each plan
    as the list of its FIELDS."""
    plans.record(net, prec, fuse, no_s2)
    q = prec == "int8"
    return {str(i): [p[k] for k in FIELDS] for i in range(net.n) if (p := net.tc_plan(i, quantized=q))}


def main():
    import tempfile
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "tc_plans.json")
    for k in PLAN_ENV:
        os.environ.pop(k, None)
    wd = tempfile.mkdtemp()
    name, sms = device()
    rec = {"size": plans.SIZE, "batch": plans.BATCH, "device": name, "sms": sms, "fields": list(FIELDS), "cases": []}
    nets = {}
    for model, prec, fuse, no_s2 in plans.cases():
        key = (model, prec == "int8")
        if key not in nets:
            nets.clear()
            nets[key] = plans.load(model, prec, wd)
        r = record(nets[key], prec, fuse, no_s2)
        rec["cases"].append(dict(model=model, prec=prec, fuse=fuse, no_s2=no_s2, plans=r))
        print(model, prec, fuse, no_s2, len(r), flush=True)
    with open(out, "w") as f:
        json.dump(rec, f, indent=None, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
