"""Records tests/golden/engine_plans*.json: the op sequence and buffer facts of the engine the library builds for every model
of cfgs.MODELS (full width, 128 x 128, batch 2, seeded synthetic weights), in every precision the model supports, with fusion
off and on, and with and without YB_NO_STEM_S2_FUSE.  The precisions "int8" and "int8_gpu" are the CPU build's and the GPU
build's INT8 rules (`quantized` = 1 and 2) on the same quantized parse.  Needs a GPU:
    python tests/golden/make_engine_plans.py [OUT_DIR]

Per case it stores the (layer, op kind) list of the profile, the engine's `launches`, `tc_layers` and `act_bytes`, the
layers whose fetch_layer raises, and `placed_only`: the engine allocated only the outputs some op writes (cases recorded
before it did lack the flag).  tests/test_gpu_engine_plan.py rebuilds the same cases with record() and compares.
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
PRECS = ("bf16", "fp32", "int8", "int8_gpu")
# the pinned files (suffix of the stem) and the precisions each holds: the GPU INT8 rule's cases were recorded after the others,
# and each file is written whole
GOLDEN = {"": PRECS[:3], "_int8_gpu": PRECS[3:]}


def model_files(model, workdir):
    secs = cfgs.MODELS[model](SIZE, SIZE)
    cfg = os.path.join(workdir, f"plan_{model}.cfg")
    wts = os.path.join(workdir, f"plan_{model}.weights")
    if not os.path.exists(wts):
        cfgs.write_cfg(secs, cfg)
        cfgs.write_weights(secs, wts, seed=WSEED)
    return cfg, wts


def precisions(model):
    """bf16 and fp32 for every model; the two INT8 rules for the models that ship input calibration."""
    net_opts = cfgs.MODELS[model](SIZE, SIZE)[0][1]
    return PRECS if "input_calibration" in net_opts else PRECS[:2]


def rule(prec):
    """the INT8 rule (the `quantized` argument of a forward call) a precision runs under"""
    return {"int8": 1, "int8_gpu": 2}.get(prec, 0)


def cases():
    # YB_NO_STEM_S2_FUSE only switches off k_stem_s2_tc, which runs in bf16 networks: the GPU INT8 rule's cases, which keep f32
    # activations, record the default alone
    return [(m, p, fuse, no_s2) for m in cfgs.MODELS for p in precisions(m) for fuse in (0, 1)
            for no_s2 in ((0,) if p == "int8_gpu" else (0, 1))]


def load_pinned(stem):
    """the recording of every pinned file of `stem` ("engine_plans" or "tc_plans"): their common header and all their cases"""
    rec = None
    for sfx in GOLDEN:
        with open(os.path.join(HERE, f"{stem}{sfx}.json")) as f:
            part = json.load(f)
        if rec is None:
            rec = part
            continue
        assert {k: v for k, v in part.items() if k != "cases"} == {k: v for k, v in rec.items() if k != "cases"}, sfx
        rec["cases"] += part["cases"]
    return rec


def write_pinned(out_dir, stem, header, record_case):
    """records every file of `stem` into out_dir: the header and, per case of the file's precisions, the case's key and
    record_case(net, prec, fuse, no_s2), net being the case's network (one per model and parse)"""
    import tempfile
    wd = tempfile.mkdtemp()
    for sfx, precs in GOLDEN.items():
        rec = dict(header, cases=[])
        nets = {}
        for model, prec, fuse, no_s2 in cases():
            if prec not in precs:
                continue
            key = (model, rule(prec) > 0)
            if key not in nets:
                nets.clear()
                nets[key] = load(model, prec, wd)
            rec["cases"].append(dict(model=model, prec=prec, fuse=fuse, no_s2=no_s2, **record_case(nets[key], prec, fuse, no_s2)))
            print(stem + sfx, model, prec, fuse, no_s2, flush=True)
        with open(os.path.join(out_dir, f"{stem}{sfx}.json"), "w") as f:
            json.dump(rec, f, indent=None, separators=(",", ":"))
            f.write("\n")


def load(model, prec, workdir):
    import yolo2_light_b200 as yb
    cfg, wts = model_files(model, workdir)
    return yb.load_network(cfg, wts, batch=BATCH, quantized=int(rule(prec) > 0))


def record(net, prec, fuse, no_s2):
    """Builds and runs the engine of one case on `net` (loaded by load() for this precision) and returns its facts."""
    import yolo2_light_b200 as yb
    q = rule(prec)
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
    out = sys.argv[1] if len(sys.argv) > 1 else HERE
    write_pinned(out, "engine_plans", {"size": SIZE, "batch": BATCH},
                 lambda net, prec, fuse, no_s2: dict(record(net, prec, fuse, no_s2), placed_only=1))


if __name__ == "__main__":
    main()
