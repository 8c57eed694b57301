"""The session collect restatement (``tests/session_collect_oracle.py``) and this repository's host engine against the
reference's own rows (``tests/golden/session_collect_cases.json``), the release rule, and which `collect_window` calls
carry the session plan.  CPU only."""

import json
import os
from datetime import datetime, timedelta, timezone

import pytest

from oracle.streams import rows_digest
from tests import session_collect_oracle as sc

S, A = sc.S, sc.A
EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)


def _host_rows(spec, steps, into):
    """The host engine's down / late / meta rows of a `collect_window` over `SessionWindower` fed the steps: values are
    the handles (dict: ``dict_value``), a frozen system clock per step.  Notify steps are not replayed here."""
    import bytewax_b200.operators as op
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource, run_main

    ts_of = {}
    items = []
    for st in steps:
        for k, t, v in zip(st[2], st[3], st[4]):
            ts_of[v] = t
            items.append((str(k), v if into != "dict" else sc.dict_value(v)))
    handle = (lambda v: v[1]) if into == "dict" else (lambda v: v)
    wait = timedelta.max if spec["wait_us"] == sc.WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    now = EPOCH + timedelta(microseconds=steps[0][1])
    clock = win.EventClock(lambda v: EPOCH + timedelta(microseconds=ts_of[handle(v)]), wait_for_system_duration=wait, now_getter=lambda: now)
    down, late, meta = [], [], []
    flow = Dataflow("h")
    keyed = op.key_on("k", op.input("in", flow, TestingSource(items, batch_size=len(items))), lambda kv: kv[0])
    wo = win.collect_window("c", op.map_value("v", keyed, lambda kv: kv[1]), clock, win.SessionWindower(gap=timedelta(microseconds=spec["gap_us"])),
                            into={"list": list, "set": set, "dict": dict}[into], ordered=spec["ordered"])
    op.output("d", wo.down, TestingSink(down))
    op.output("l", wo.late, TestingSink(late))
    op.output("m", wo.meta, TestingSink(meta))
    run_main(flow, gpu=False)
    return down, late, meta


def _one_batch(seed):
    """A seeded stream folded into one activation with a frozen clock, so the host engine sees exactly its items."""
    spec, steps = sc.seeded_steps(seed, moving=False)
    batches = [s for s in steps if s[0] == "batch"]
    one = ["batch", batches[0][1], [k for s in batches for k in s[2]], [t for s in batches for t in s[3]], [v for s in batches for v in s[4]]]
    return spec, [one]


@pytest.mark.parametrize("into", sc.INTOS)
@pytest.mark.parametrize("seed", list(range(0, 48, 3)))
def test_oracle_matches_host_engine(seed, into):
    spec, steps = _one_batch(seed)
    acts, _rel = sc.run_session_collect(spec, steps)
    rows = [r for a in acts for r in a]
    vo = sc.dict_value if into == "dict" else (lambda h: h)
    want_down = [(str(r[0]), (r[1], sc.container(into, r[3][0], r[3][1], vo))) for r in rows if r[2] == "E"]
    want_late = [(str(r[0]), (-1, vo(r[3]))) for r in rows if r[2] == "L"]
    want_meta = [(str(r[0]), (r[1], r[3][0], r[3][1], set(r[3][2]))) for r in rows if r[2] == "M"]
    down, late, meta = _host_rows(spec, steps, into)

    def us(d):
        delta = d - EPOCH
        return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds

    def order(c):
        return list(c.items()) if isinstance(c, dict) else list(c)

    assert [(k, w, order(c)) for k, (w, c) in down] == [(k, w, order(c)) for k, (w, c) in want_down]
    assert late == want_late
    assert [(k, (w, us(m.open_time), us(m.close_time), m.merged_ids)) for k, (w, m) in meta] == [(k, x) for k, x in want_meta]


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "session_collect_cases.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _case_names():
    with open(GOLDEN) as f:
        return sorted(json.load(f)["cases"])


def _seeded_names():
    with open(GOLDEN) as f:
        return sorted(json.load(f)["seeded"])


@pytest.mark.parametrize("name", _case_names())
def test_oracle_matches_golden_case(golden, name):
    c = golden["cases"][name]
    st = {}
    acts, _ = sc.run_session_collect(c["spec"], c["steps"], stats=st)
    assert sc.golden_rows(c["into"], acts) == c["acts"]
    assert (st["merges"] > 0) == (c["merges"] > 0)


@pytest.mark.parametrize("name", _seeded_names())
def test_oracle_matches_golden_digest(golden, name):
    seed, into = name[len("seed_"):].split("/")
    spec, steps = sc.seeded_steps(int(seed), moving=int(seed) % 3 != 0)
    acts, _ = sc.run_session_collect(spec, steps)
    rows = sc.golden_rows(into, acts)
    assert [len(a) for a in rows] == golden["seeded"][name]["rows"]
    assert rows_digest(rows) == golden["seeded"][name]["sha256"]


def _host_builder(c, now):
    """This repository's own `collect_window` logic (the host engine's), built as the reference's is by the generator."""
    import bytewax_b200.operators as op
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSource

    def find(flow):
        stack = list(flow.substeps)
        while stack:
            step = stack.pop(0)
            if getattr(step, "builder", None) is not None and hasattr(step.builder, "_gpu_session_collect_plan"):
                return step
            stack = list(getattr(step, "substeps", None) or []) + stack
        raise LookupError("no stateful_batch step")

    return sc.builder_of(win, op, Dataflow, TestingSource, find, c["spec"], c["steps"], c["into"], now, _dt)


def _dt(t):
    return EPOCH + timedelta(microseconds=t)


def _us(d):
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


@pytest.mark.parametrize("name", _case_names())
def test_host_engine_matches_golden_case(golden, name):
    c = golden["cases"][name]
    now = [_dt(c["steps"][0][1])]
    acts, merges = sc.drive(_host_builder(c, now), c["steps"], now, _us, _dt, c["into"])
    assert acts == c["acts"] and merges == c["merges"]


@pytest.mark.parametrize("name", _seeded_names())
def test_host_engine_matches_golden_digest(golden, name):
    seed, into = name[len("seed_"):].split("/")
    spec, steps = sc.seeded_steps(int(seed), moving=int(seed) % 3 != 0)
    c = dict(spec=spec, steps=steps, into=into)
    now = [_dt(steps[0][1])]
    acts, _ = sc.drive(_host_builder(c, now), steps, now, _us, _dt, into)
    assert rows_digest(acts) == golden["seeded"][name]["sha256"]


def test_golden_sets_catch_a_flat_rebuild(golden):
    """In the golden set cases the generator marked, some merged session's set as the reference built it iterates unlike
    a flat replay of its values, so a flat rebuild on the device's data would fail the golden tests."""
    assert len(golden["set_flat_differs"]) >= 3
    for name in golden["set_flat_differs"]:
        c = golden["cases"][name + "/set"]
        acts, _ = sc.run_session_collect(c["spec"], c["steps"])
        flat_rows = sc.golden_rows("set", [[r if r[2] != "E" else r[:3] + [[r[3][0], []]] for r in a] for a in acts])  # no intervals
        assert flat_rows != c["acts"], name


@pytest.mark.parametrize("seed", list(sc.SEEDED))
def test_release_rule_and_ordered_never_merges(seed):
    spec, steps = sc.seeded_steps(seed, moving=seed % 3 != 0)
    st = {}
    acts, rel = sc.run_session_collect(spec, steps, stats=st)
    assert not (spec["ordered"] and st["merges"])
    # every handle released exactly once, in the call whose rows carry it (its session's E row, or its late row)
    flat = [h for r in rel for h in r]
    every = [v for s in steps if s[0] == "batch" for v in s[4]]
    assert sorted(flat) == sorted(every)
    for rows, r in zip(acts, rel):
        carried = sorted([h for x in rows if x[2] == "E" for h in x[3][0]] + [x[3] for x in rows if x[2] == "L"])
        assert carried == r


def _plans(into=list, ordered=True, windower=None, clock=None):
    import bytewax_b200.operators as op
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.operators import windowing as W
    from bytewax_b200.testing import TestingSource

    windower = windower or W.SessionWindower(gap=timedelta(seconds=5))
    clock = clock or W.EventClock(lambda v: EPOCH, wait_for_system_duration=timedelta(seconds=1))
    flow = Dataflow("plan")
    up = op.key_on("k", op.input("in", flow, TestingSource([])), lambda _v: "k")
    W.collect_window("collect", up, clock, windower, into=into, ordered=ordered)
    found = {"_gpu_plan": [], "_gpu_session_collect_plan": []}

    def walk(step):
        b = getattr(step, "builder", None)
        for attr, got in found.items():
            if b is not None and getattr(b, attr, None) is not None:
                got.append(getattr(b, attr))
        for sub in getattr(step, "substeps", []) or []:
            walk(sub)

    for s in flow.substeps:
        walk(s)
    return found


@pytest.mark.parametrize("into", [list, set, dict])
@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("clock", ["event", "system"])
def test_session_plan_on_its_own_attribute(into, ordered, clock):
    from bytewax_b200 import engine
    from bytewax_b200.operators import windowing as W

    c = W.SystemClock() if clock == "system" else W.EventClock(lambda v: EPOCH, wait_for_system_duration=timedelta.max)
    found = _plans(into, ordered, clock=c)
    assert found["_gpu_plan"] == []
    (plan,) = found["_gpu_session_collect_plan"]
    assert isinstance(plan, W.GpuSessionCollectWindowPlan) and plan.into is into and plan.ordered is ordered and plan.clock is c
    assert isinstance(engine._gpu_step_for("s", plan), engine._GpuSessionCollectWindowStep)
    assert W._collect_window_plan("c", c, plan.windower, into, ordered) is None


def test_no_session_plan_off_the_device():
    from bytewax_b200.operators import windowing as W

    class MyList(list):
        pass

    align = datetime(2022, 1, 1, tzinfo=timezone.utc)
    assert _plans(MyList)["_gpu_session_collect_plan"] == []
    assert _plans(clock=W.EventClock(lambda v: align, timedelta(0), to_system_utc=lambda t: t))["_gpu_session_collect_plan"] == []
    tumbling = _plans(windower=W.TumblingWindower(length=timedelta(seconds=10), align_to=align))
    assert tumbling["_gpu_session_collect_plan"] == [] and len(tumbling["_gpu_plan"]) == 1
