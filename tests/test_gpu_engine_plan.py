"""The engine's op sequence, pinned per model, precision and fusion setting (tests/golden/engine_plans*.json, recorded with
tests/golden/make_engine_plans.py): the same ops in the same order on the same layers, the same launch and tensor-core counts.
Activation memory holds only outputs some op writes: every layer whose fetch_layer raises has no buffer, the NHWC input copy
exists only when the first op makes it, and a detection head whose [yolo] layer runs in its epilogue raises too.
Networks the op list cannot express fail when the engine is built, with the layer plan's message."""
import re
import sys

import pytest

import ybtest_util as util

sys.path.insert(0, util.GOLDEN)
import make_engine_plans as plans  # noqa: E402

pytestmark = pytest.mark.gpu

PINNED = plans.load_pinned("engine_plans")
MODELS = sorted({c["model"] for c in PINNED["cases"]})

DT_BYTES = {"f32": 4, "bf16": 2}


def _align(v, a=1024):
    return (v + a - 1) // a * a


def _freed_bytes(net, prec, case, raises):
    """Bytes of the buffers that a recorded case allocated and the current engine does not: none when the recording engine
    placed only the outputs some op writes (`placed_only`); before that, the outputs of layers that now raise (other than
    convolutions fused into the shortcut behind them, which never had one) and the NHWC input copy when a stem reads the
    caller's images."""
    if case.get("placed_only"):
        return 0
    layers = net.layers
    B = PINNED["batch"]
    exact = prec != "bf16" or any(l["type_name"] == "CONVOLUTIONAL" and l["xnor"] for l in layers)
    act = "f32" if exact else "bf16"
    freed = 0
    if case["ops"][0][1] != "input":
        freed += _align(B * (net.h + 2) * (net.w + 2) * net.c * DT_BYTES[act])
    for i in raises:
        l = layers[i]
        nxt = layers[i + 1]["type_name"] if i + 1 < len(layers) else None
        if case["fuse"] and l["type_name"] == "CONVOLUTIONAL" and nxt == "SHORTCUT":
            continue
        head = l["type_name"] == "CONVOLUTIONAL" and nxt in ("YOLO", "REGION")
        dt = "f32" if head else act
        freed += _align(B * (l["out_h"] + 2) * (l["out_w"] + 2) * _align(l["out_c"], 8) * DT_BYTES[dt])
    return freed


@pytest.mark.parametrize("model", MODELS)
def test_engine_plan_matches_pinned(model, workdir):
    cases = [c for c in PINNED["cases"] if c["model"] == model]
    assert len(cases) == len([k for k in plans.cases() if k[0] == model])
    nets = {}
    for case in cases:
        prec, fuse, no_s2 = case["prec"], case["fuse"], case["no_s2"]
        q = plans.rule(prec) > 0    # the two INT8 rules run on one quantized parse
        if q not in nets:
            nets[q] = plans.load(model, prec, workdir)
        net = nets[q]
        got = plans.record(net, prec, fuse, no_s2)
        what = (model, prec, fuse, no_s2)
        assert got["ops"] == case["ops"], what
        assert got["launches"] == case["launches"] and got["tc_layers"] == case["tc_layers"], what
        # the [yolo] layers with no op of their own are written by their head's epilogue: the head now raises
        ops_layers = {li for li, _ in case["ops"]}
        fused_heads = {i - 1 for i, l in enumerate(net.layers) if l["type_name"] == "YOLO" and i not in ops_layers}
        assert set(got["raises"]) == set(case["raises"]) | fused_heads, what
        assert got["act_bytes"] == case["act_bytes"] - _freed_bytes(net, prec, case, got["raises"]), what


def _edit(descs, i, **fields):
    for k, v in fields.items():
        setattr(descs[i], k, v)
    return descs


# (case, model, edit of its layer descriptors, message)
REJECTED = [
    ("reverse_upsample", "tiny64", lambda d: _edit(d, 19, reverse=1), "engine: reverse upsample (downsample) is not supported"),
    ("reverse_reorg", "v2voc32", lambda d: _edit(d, 27, reverse=1), "engine: reverse reorg is not supported"),
    ("conv_input_shape", "tiny64", lambda d: _edit(d, 2, h=31, w=31), "engine: conv input shape mismatch"),
    ("upsample_behind_yolo", "tiny64", lambda d: d[:17] + [d[19]], "engine: layer 17 has no image input"),
    ("route_sizes", "tiny64", lambda d: _edit(d, 20, out_h=0),
     "engine: route over layers of different spatial size is not supported"),
]


@pytest.mark.parametrize("case,model,edit,msg", REJECTED, ids=[r[0] for r in REJECTED])
def test_engine_rejects_unsupported_network(case, model, edit, msg, workdir):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files(model, workdir)
    src = yb.load_network(cfg, wts, batch=2)
    net = yb.network_from_layers(edit([src.layer_desc(i) for i in range(src.n)]), 2, src.h, src.w, src.c)
    with pytest.raises(yb.YbError, match=re.escape(msg)):
        net.predict(util.images(model, 2))
