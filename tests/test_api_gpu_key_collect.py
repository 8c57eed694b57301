"""`collect` flows with the CUDA path enabled (run_main(..., gpu=True)): an `int` max_size hands the step to K13
(`bw_kcollect_*`); its rows must equal the host engine's.  -m gpu."""

import json
import os
import random
from datetime import timedelta

import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.errors import BytewaxRuntimeError  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402
from tests import key_collect_oracle as ko  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "key_collect_cases.json")


@pytest.fixture
def k13_steps(monkeypatch):
    """Records every collect step that ran an activation on the device, to check that the CUDA path really ran."""
    made = []
    orig = engine._GpuCollectStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert self.jwin is not None
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuCollectStep, "on_epoch", on_epoch)
    return made


def _both(build, **kw):
    outs = []
    for gpu in (False, True):
        flow, out = build()
        run_main(flow, gpu=gpu, **kw)
        outs.append(out)
    return outs


def test_reference_test_collect(k13_steps):
    # pytests/operators/test_collect.py::test_collect
    def build():
        out = []
        flow = Dataflow("test_df")
        s = op.input("inp", flow, TestingSource(list(range(10))))
        s = op.key_on("key", s, lambda _x: "ALL")
        s = op.collect("collect", s, timedelta(seconds=10), 3)
        op.output("out", s, TestingSink(out))
        return flow, out

    host, gpu = _both(build)
    assert host == gpu == [("ALL", [0, 1, 2]), ("ALL", [3, 4, 5]), ("ALL", [6, 7, 8]), ("ALL", [9])]
    assert k13_steps and all(s.resort for s in k13_steps)


def test_docstring_example(k13_steps):
    source = [{"key": "ab"[i % 2], "val": i + 1} for i in range(8)]

    def build():
        out = []
        flow = Dataflow("collect_eg")
        keyed = op.key_on("key", op.input("nums", flow, TestingSource(source)), lambda x: x["key"])
        op.output("out", op.collect("collect", keyed, timedelta(seconds=1), max_size=2), TestingSink(out))
        return flow, out

    host, gpu = _both(build)
    assert host == gpu == [("a", [source[0], source[2]]), ("b", [source[1], source[3]]), ("a", [source[4], source[6]]),
                           ("b", [source[5], source[7]])]
    assert k13_steps


@pytest.mark.parametrize("workers", [1, 2])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_seeded_flows(k13_steps, workers, seed):
    rnd = random.Random(seed)
    keys = [str(rnd.randrange(10**rnd.randrange(1, 6))) for _ in range(40)] + ["a", "", "007", "é"]
    items = [(rnd.choice(keys), {"i": i}) for i in range(3000)]
    max_size = [1, 3, 64, 0, 2**70][seed % 5]
    batch_size = rnd.choice([7, 100, 1000])

    def build():
        out = []
        flow = Dataflow("df")
        s = op.input("in", flow, TestingSource(items, batch_size=batch_size))
        s = op.key_on("key", op.map("m", s, lambda x: x), lambda x: x[0])
        s = op.map_value("v", s, lambda x: x[1])
        op.output("out", op.collect("collect", s, timedelta(seconds=30), max_size), TestingSink(out))
        return flow, out

    flow, host = build()
    run_main(flow)
    flow, gpu = build()
    engine._Run(flow, workers, None, True).run() if workers > 1 else run_main(flow, gpu=True)
    if workers == 1:
        assert gpu == host
    else:  # two workers interleave their rows: each key's lists, in order, are the host's
        per_key = lambda rows: {k: [v for kk, v in rows if kk == k] for k, _ in rows}  # noqa: E731
        assert per_key(gpu) == per_key(host) and len(gpu) == len(host)
    assert k13_steps


def test_overflowing_first_batch_goes_to_the_host(k13_steps):
    """`now + timeout` past datetime.max in the step's first batch: the host logic runs it and raises its own error."""

    def build():
        out = []
        flow = Dataflow("df")
        s = op.key_on("key", op.input("in", flow, TestingSource([1, 2, 3])), lambda _x: "k")
        op.output("out", op.collect("collect", s, timedelta.max, 2), TestingSink(out))
        return flow, out

    errors = []
    for gpu in (False, True):
        flow, _out = build()
        with pytest.raises(BytewaxRuntimeError) as ei:
            run_main(flow, gpu=gpu)
        errors.append(ei.value)
        assert isinstance(ei.value.__cause__, OverflowError)
    assert str(errors[0]) == str(errors[1]) and not k13_steps


def _drive_step(case, monkeypatch):
    """The golden case through `_GpuCollectStep` itself, the way the engine's activation loop calls it
    (engine._Run._run_stateful): a stepping `_get_system_utc` and the matching activation `now`."""
    from bytewax_b200.operators import GpuCollectPlan

    clock = [None]
    monkeypatch.setattr(op, "_get_system_utc", lambda: clock[0])
    step = engine._GpuCollectStep("df.collect", GpuCollectPlan(timedelta(microseconds=case["timeout_us"]),
                                                                max(1, min(case["max_size"], 2**64 - 1))))
    acts, last_out = [], 0
    try:
        for now, batches in case["steps"]:
            clock[0] = engine._dt(now)
            ready = {}
            for epoch, items in batches:
                ready.setdefault(epoch, []).extend(items)
            epochs = sorted(set(ready) | ({last_out} if last_out else set()))
            act = []
            acts.append(act)
            for e in epochs:
                if ready.get(e):
                    try:
                        act.append(["B", e, [[k, v] for k, v in step.on_epoch(e, [tuple(i) for i in ready[e]])]])
                    except (engine._GpuPlanUnfit, OverflowError):
                        act.append(["raises", "OverflowError"])
                        return acts, step
                act.append(["N", e, [[k, v] for k, v in step.on_notify(clock[0])]])
            if epochs:
                last_out = epochs[-1]
            act[:] = [c for c in act if c[2]]
        acts.append([c for c in [["E", None, [[k, v] for k, v in step.on_eof()]]] if c[2]])
        return acts, step
    finally:
        step.release()


with open(GOLDEN) as _f:
    _CASES = json.load(_f)["cases"]


@pytest.mark.parametrize("name", sorted(_CASES))
def test_step_under_a_stepping_clock(monkeypatch, name):
    case = _CASES[name]
    assert _drive_step(case, monkeypatch)[0] == case["rows"]


def test_later_overflow_names_the_step(monkeypatch):
    case = _CASES["timeout_at_past_utc_max"]
    with pytest.raises(OverflowError, match="step 'df.collect'"):
        from bytewax_b200.operators import GpuCollectPlan

        clock = [engine._dt(case["steps"][0][0])]
        monkeypatch.setattr(op, "_get_system_utc", lambda: clock[0])
        step = engine._GpuCollectStep("df.collect", GpuCollectPlan(timedelta(microseconds=case["timeout_us"]), 3))
        try:
            step.on_epoch(1, [("a", 1)])
            clock[0] = engine._dt(case["steps"][1][0])
            step.on_epoch(2, [("a", 2)])
        finally:
            step.release()


@pytest.mark.parametrize("seed", [0, 9, 13, 22, 31])
def test_seeded_step_matches_oracle(monkeypatch, seed):
    case = ko.seeded_case(seed, n_keys=200, steps=12, per_step=400)
    assert _drive_step(case, monkeypatch)[0] == ko.run_oracle(case)
