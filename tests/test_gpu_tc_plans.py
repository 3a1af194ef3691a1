"""The tensor-core plans, pinned per model, precision and fusion setting (tests/golden/tc_plans*.json, recorded with
tests/golden/make_tc_plans.py): every layer with a plan keeps its kernel, kind, tile shape, filter tile width, resident filter
matrix, ring depth, K-blocks per stage, grid, work items, TMA epilogue, row shift and output pitch.  The filter tile width and
the grid depend on the SM count: the comparison needs a card with the SM count of the recording."""
import sys

import pytest

import ybtest_util as util

sys.path.insert(0, util.GOLDEN)
import make_engine_plans as plans  # noqa: E402
import make_tc_plans as tc_plans  # noqa: E402

pytestmark = pytest.mark.gpu

PINNED = plans.load_pinned("tc_plans")
MODELS = sorted({c["model"] for c in PINNED["cases"]})


@pytest.mark.parametrize("model", MODELS)
def test_tc_plans_match_pinned(model, workdir, monkeypatch):
    name, sms = tc_plans.device()
    if sms != PINNED["sms"]:
        pytest.skip(f"plans recorded on a {PINNED['device']} ({PINNED['sms']} SMs), this is a {name} ({sms} SMs)")
    assert PINNED["fields"] == list(tc_plans.FIELDS)
    for k in tc_plans.PLAN_ENV:
        monkeypatch.delenv(k, raising=False)
    cases = [c for c in PINNED["cases"] if c["model"] == model]
    assert len(cases) == len([k for k in plans.cases() if k[0] == model])
    nets = {}
    for case in cases:
        prec, fuse, no_s2 = case["prec"], case["fuse"], case["no_s2"]
        q = plans.rule(prec) > 0    # the two INT8 rules run on one quantized parse
        if q not in nets:
            nets[q] = plans.load(model, prec, workdir)
        got = tc_plans.record(nets[q], prec, fuse, no_s2)
        what = (model, prec, fuse, no_s2)
        assert sorted(got, key=int) == sorted(case["plans"], key=int), what
        for layer, fields in case["plans"].items():
            assert dict(zip(PINNED["fields"], got[layer])) == dict(zip(PINNED["fields"], fields)), (what, int(layer))
