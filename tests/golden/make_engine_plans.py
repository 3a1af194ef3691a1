"""Records tests/golden/engine_plans.json: the op sequence and buffer facts of the engine the library builds for every model
of cfgs.MODELS (full width, 128 x 128, batch 2, seeded synthetic weights), in every precision the model supports, with fusion
off and on, and with and without YB_NO_STEM_S2_FUSE.  Needs a GPU:
    python tests/golden/make_engine_plans.py [OUT.json]

Per case it stores the (layer, op kind) list of the profile, the engine's `launches`, `tc_layers` and `act_bytes`, and the
layers whose fetch_layer raises.  tests/test_gpu_engine_plan.py rebuilds the same cases with record() and compares.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from yolo2_light_b200 import cfgs  # noqa: E402

SIZE, BATCH, WSEED, XSEED = 128, 2, 91, 92
PRECS = ("bf16", "fp32", "int8")


def model_files(model, workdir):
    secs = cfgs.MODELS[model](SIZE, SIZE)
    cfg = os.path.join(workdir, f"plan_{model}.cfg")
    wts = os.path.join(workdir, f"plan_{model}.weights")
    if not os.path.exists(wts):
        cfgs.write_cfg(secs, cfg)
        cfgs.write_weights(secs, wts, seed=WSEED)
    return cfg, wts


def precisions(model):
    """bf16 and fp32 for every model; the quantized rule for the models that ship input calibration."""
    net_opts = cfgs.MODELS[model](SIZE, SIZE)[0][1]
    return PRECS if "input_calibration" in net_opts else PRECS[:2]


def cases():
    return [(m, p, fuse, no_s2) for m in cfgs.MODELS for p in precisions(m) for fuse in (0, 1) for no_s2 in (0, 1)]


def load(model, prec, workdir):
    import yolo2_light_b200 as yb
    cfg, wts = model_files(model, workdir)
    return yb.load_network(cfg, wts, batch=BATCH, quantized=int(prec == "int8"))


def record(net, prec, fuse, no_s2):
    """Builds and runs the engine of one case on `net` (loaded by load() for this precision) and returns its facts."""
    import yolo2_light_b200 as yb
    q = prec == "int8"
    net.set_precision(yb.YB_PREC_FP32 if prec == "fp32" else yb.YB_PREC_BF16_TC)
    net.set_option("fuse", fuse)   # drops the engine: the next call builds one under the switches below
    old = os.environ.pop("YB_NO_STEM_S2_FUSE", None)
    if no_s2:
        os.environ["YB_NO_STEM_S2_FUSE"] = "1"
    try:
        net.predict(cfgs.synthetic_images(BATCH, 3, SIZE, SIZE, seed=XSEED), quantized=q)
    finally:
        os.environ.pop("YB_NO_STEM_S2_FUSE", None)
        if old is not None:
            os.environ["YB_NO_STEM_S2_FUSE"] = old
    raises = []
    for i in range(net.n):
        try:
            net.fetch_layer(i, quantized=q)
        except yb.YbError:
            raises.append(i)
    return {"ops": [[li, kind] for li, kind, _ in net.profile(quantized=q)],
            "launches": net.get_info("launches", quantized=q),
            "tc_layers": net.get_info("tc_layers", quantized=q),
            "act_bytes": net.get_info("act_bytes", quantized=q),
            "raises": raises}


def main():
    import tempfile
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "engine_plans.json")
    wd = tempfile.mkdtemp()
    rec = {"size": SIZE, "batch": BATCH, "cases": []}
    nets = {}
    for model, prec, fuse, no_s2 in cases():
        key = (model, prec == "int8")
        if key not in nets:
            nets.clear()
            nets[key] = load(model, prec, wd)
        r = record(nets[key], prec, fuse, no_s2)
        rec["cases"].append(dict(model=model, prec=prec, fuse=fuse, no_s2=no_s2, **r))
        print(model, prec, fuse, no_s2, r["launches"], r["tc_layers"], r["act_bytes"], r["raises"], flush=True)
    with open(out, "w") as f:
        json.dump(rec, f, indent=None, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
