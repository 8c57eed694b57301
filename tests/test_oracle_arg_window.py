"""The CPU restatement of `max_window` / `min_window` with ``by=`` (tests/arg_window_oracle.py) against the reference's
own rows (tests/golden/arg_window_cases.json, tools/gen_arg_window_golden.py), its release rule, and which plan the
operators attach.  No GPU."""

import json
import math
import os
from datetime import datetime, timedelta, timezone

import pytest

from oracle.streams import rows_digest
from tests import arg_window_oracle as aw

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "arg_window_cases.json")))


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_oracle_matches_reference_case(name):
    case = GOLDEN["cases"][name]
    acts, _ = aw.run_arg_window(case["spec"], case["steps"])
    assert acts == case["acts"]


@pytest.mark.parametrize("seed", list(aw.SEEDED))
def test_oracle_matches_reference_digest(seed):
    spec, steps = aw.seeded_steps(seed, moving=seed % 3 != 1)
    acts, _ = aw.run_arg_window(spec, steps)
    want = GOLDEN["seeded"][f"seed_{seed}"]
    assert [len(a) for a in acts] == want["rows"]
    assert rows_digest(acts) == want["sha256"]


def test_golden_covers_the_edges():
    names = set(GOLDEN["cases"])
    for want in ("signed_zero_ties_max", "nan_first_max", "nan_later_min", "inf_subnormal_max", "i64_extremes_min",
                 "sliding_pick_in_some_windows", "late_with_wait", "moving_clock_notify", "discard_and_reopen",
                 "merge_survivor_wins_tie_with_later_pick", "value_into_merged_away_session", "merge_chain_one_call",
                 "session_eof_near_utc_max"):
        assert want in names
    # NaN and -0.0 survive the JSON round trip
    bys = [aw.dec(b) for c in GOLDEN["cases"].values() for s in c["steps"] if s[0] == "batch" for b in s[4]]
    assert any(isinstance(b, float) and math.isnan(b) for b in bys)
    assert any(isinstance(b, float) and b == 0 and math.copysign(1, b) < 0 for b in bys)


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_release_rule(name):
    """Every handle is released exactly once, in the call after whose rows no window names it any more; a handle named
    by a row is never released before that row's call."""
    case = GOLDEN["cases"][name]
    acts, released = aw.run_arg_window(case["spec"], case["steps"])
    got = [h for r in released for h in r]
    every = [h for s in case["steps"] if s[0] == "batch" for h in s[5]]
    assert len(got) == len(set(got))
    # sessions that close at or after UTC_MAX - gap stay open past EOF, and keep their picks (keys 22 and 24 here)
    assert set(every) - set(got) == ({0, 2} if name == "session_eof_near_utc_max" else set())
    when = {h: i for i, r in enumerate(released) for h in r}
    for i, act in enumerate(acts):
        for row in act:
            if row[2] in ("E", "L"):
                assert when[row[3]] >= i, (name, row)
    # a late item and a value that is the pick of none of its windows go in the call that received them
    for i, s in enumerate(case["steps"]):
        if s[0] != "batch":
            continue
        for row in acts[i]:
            if row[2] == "L":
                assert row[3] in released[i]


def test_release_rule_seeded():
    for seed in aw.SEEDED:
        spec, steps = aw.seeded_steps(seed)
        _, released = aw.run_arg_window(spec, steps)
        got = [h for r in released for h in r]
        assert sorted(got) == [h for s in steps if s[0] == "batch" for h in s[5]]


# --- plan routing ------------------------------------------------------------------------------------------------------
ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)


def _plan(fn_name, clock, windower, **kw):
    import bytewax_b200.operators as op
    import bytewax_b200.operators.windowing as W
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSource

    flow = Dataflow("p")
    s = op.key_on("k", op.input("in", flow, TestingSource([])), lambda e: "a")
    getattr(W, fn_name)("w", s, clock, windower, **kw)
    found = []

    def walk(step):
        b = getattr(step, "builder", None)
        if b is not None and getattr(b, "_gpu_plan", None) is not None:
            found.append(b._gpu_plan)
        for sub in getattr(step, "substeps", []) or []:
            walk(sub)

    for st in flow.substeps:
        walk(st)
    assert len(found) <= 1
    return found[0] if found else None


def _windowers():
    import bytewax_b200.operators.windowing as W

    return [W.TumblingWindower(length=timedelta(seconds=10), align_to=ALIGN),
            W.SlidingWindower(length=timedelta(seconds=10), offset=timedelta(seconds=5), align_to=ALIGN),
            W.SessionWindower(gap=timedelta(seconds=2))]


def _clocks():
    import bytewax_b200.operators.windowing as W

    return [W.EventClock(lambda e: e["t"], wait_for_system_duration=timedelta(0)), W.SystemClock()]


@pytest.mark.parametrize("fn_name", ["max_window", "min_window"])
def test_by_attaches_arg_window_plan(fn_name):
    import bytewax_b200.operators.windowing as W

    by = lambda e: e["val"]  # noqa: E731
    for windower in _windowers():
        for clock in _clocks():
            plan = _plan(fn_name, clock, windower, by=by)
            assert isinstance(plan, W.GpuArgWindowPlan)
            assert plan.extreme == fn_name[:3] and plan.by is by and plan.windower is windower and plan.clock is clock


@pytest.mark.parametrize("fn_name", ["max_window", "min_window"])
def test_identity_by_keeps_fold_plan(fn_name):
    import bytewax_b200.operators.windowing as W

    for windower in _windowers():
        plan = _plan(fn_name, _clocks()[0], windower)
        assert isinstance(plan, W.GpuFoldPlan) and plan.reduction == fn_name[:3]


@pytest.mark.parametrize("fn_name", ["max_window", "min_window"])
def test_custom_to_system_utc_stays_on_host(fn_name):
    import bytewax_b200.operators.windowing as W

    clock = W.EventClock(lambda e: e["t"], wait_for_system_duration=timedelta(0), to_system_utc=lambda t: t)
    for windower in _windowers():
        assert _plan(fn_name, clock, windower, by=lambda e: e["val"]) is None


def test_engine_routes_arg_window_plan():
    import bytewax_b200.engine as E
    import bytewax_b200.operators.windowing as W

    for windower in _windowers():
        step = E._gpu_step_for("s", W.GpuArgWindowPlan("max", lambda e: e, _clocks()[0], windower))
        assert type(step) is E._GpuArgWindowStep
        assert (step.gap_us is not None) == isinstance(windower, W.SessionWindower)


def test_by_type_rules_before_and_after_the_first_batch():
    """In the first batch a `by` the device cannot carry sends the step to the host logic (_GpuPlanUnfit); afterwards
    the same raises a TypeError naming the step."""
    import bytewax_b200.engine as E
    import bytewax_b200.operators.windowing as W

    plan = W.GpuArgWindowPlan("max", lambda e: e["val"], _clocks()[0], _windowers()[0])
    bad = [{"val": "x"}, {"val": True}, {"val": 1 << 63}, {"val": None}, {}]
    for v in bad:
        step = E._gpu_step_for("s", plan)
        with pytest.raises(E._GpuPlanUnfit):
            step._by(v)
    step = E._gpu_step_for("s", plan)
    assert step._by({"val": 3}) == 3
    with pytest.raises(E._GpuPlanUnfit):
        step._by({"val": 2.5})  # int then float
    step.jwin = object()  # (as if the device step existed: no longer the first batch)
    for v in bad + [{"val": 2.5}]:
        with pytest.raises(TypeError, match="'s'"):
            step._by(v)
    assert step._by({"val": -(1 << 63)}) == -(1 << 63)
