"""Records tests/golden/tc_plans*.json: the tensor-core plan (Network.tc_plan) of every layer that has one, for every case of
make_engine_plans.cases() (every model of cfgs.MODELS, precision and fusion setting; 128 x 128, batch 2), in the files of
make_engine_plans.GOLDEN.  Needs a GPU:
    python tests/golden/make_tc_plans.py [OUT_DIR]

A plan's filter tile width and grid depend on the SM count, so the file names the card it was recorded on and its SM count;
tests/test_gpu_tc_plans.py rebuilds the same cases and compares on a card with the same SM count.
"""
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
    q = plans.rule(prec)
    return {str(i): [p[k] for k in FIELDS] for i in range(net.n) if (p := net.tc_plan(i, quantized=q))}


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else HERE
    for k in PLAN_ENV:
        os.environ.pop(k, None)
    name, sms = device()
    header = {"size": plans.SIZE, "batch": plans.BATCH, "device": name, "sms": sms, "fields": list(FIELDS)}
    plans.write_pinned(out, "tc_plans", header, lambda net, prec, fuse, no_s2: {"plans": record(net, prec, fuse, no_s2)})


if __name__ == "__main__":
    main()
