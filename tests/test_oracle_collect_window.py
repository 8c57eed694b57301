"""The `collect_window` restatement (tests/collect_window_oracle.py) against rows of the reference's own, unmodified
`_WindowLogic` + `_SlidingWindowerLogic` + `_FoldWindowLogic` with the collect callbacks
(tests/golden/collect_window_cases.json, made by tools/gen_collect_window_golden.py), the handle-release rule the device
follows, and which `collect_window` calls carry a GPU plan."""

import json
import os
from datetime import datetime, timedelta, timezone

import pytest

from oracle.streams import rows_digest
from tests import collect_window_oracle as co

S, A = co.S, co.A
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "collect_window_cases.json")

with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_case_list(golden):
    want = {"reference_test_stream", "docstring_example", "sliding_indivisible_offset", "negative_window_ids",
            "late_sliding_all_windows", "close_first_opened_not_id_order", "ordered_ties_stable",
            "ordered_queue_across_activations", "ordered_notify_wakes_queue_head", "wait_forever_flush_at_eof",
            "discard_resets_watermark", "system_clock_moving_now", "near_utc_max"}
    assert want <= set(golden["cases"])


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hand_built_case(golden, name):
    case = golden["cases"][name]
    acts, _ = co.run_collect_window(case["spec"], case["steps"])
    assert acts == case["acts"]


@pytest.mark.parametrize("seed", list(co.SEEDED))
def test_seeded_digests(golden, seed):
    spec, steps = co.seeded_steps(seed, moving=seed % 3 != 0)
    acts, _ = co.run_collect_window(spec, steps)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in acts] == want["rows"]
    assert rows_digest(acts) == want["sha256"]


def test_seeded_streams_cover_every_shape():
    shapes, lates, emits = set(), 0, 0
    for seed in co.SEEDED:
        spec, steps = co.seeded_steps(seed, moving=seed % 3 != 0)
        shapes.add((spec["ordered"], spec["length_us"] == spec["offset_us"], spec["wait_us"]))
        acts, _ = co.run_collect_window(spec, steps)
        lates += sum(r[2] == "L" for a in acts for r in a)
        emits += sum(r[2] == "E" for a in acts for r in a)
    assert len(shapes) == 16 and lates > 100 and emits > 500


@pytest.mark.parametrize("seed", list(co.SEEDED))
def test_every_handle_released_once(seed):
    """Each input handle is released exactly once, by EOF at the latest, in the call that closes the last window holding
    it (a late item's: the call that received it), and no row names a handle released earlier."""
    spec, steps = co.seeded_steps(seed, moving=seed % 3 != 0)
    acts, released = co.run_collect_window(spec, steps)
    flat = [h for r in released for h in r]
    inputs = [v for st in steps if st[0] == "batch" for v in st[5]]
    assert sorted(flat) == sorted(inputs)
    gone, last_e = set(), {}
    for i, (act, rel) in enumerate(zip(acts, released)):
        for r in act:
            vals = r[3] if r[2] == "E" else ([r[3]] if r[2] == "L" else [])
            assert not gone.intersection(vals)
            for v in vals:
                last_e[v] = i
        gone.update(rel)
        for h in rel:
            assert last_e.get(h) == i  # released with the last row that carries it


def test_sliding_release_waits_for_the_highest_window():
    spec = dict(ordered=False, length_us=6 * S, offset_us=2 * S, align_us=A, wait_us=0)
    # the value at A sits in windows -2, -1, 0 ([A-4s, A+2s) ... [A, A+6s)): released when window 0 closes
    steps = [["batch", A, [1], [A], [0], [10]], ["batch", A, [1], [A + 2 * S], [0], [11]], ["batch", A, [1], [A + 4 * S], [0], [12]],
             ["batch", A, [1], [A + 6 * S], [0], [13]]]
    acts, released = co.run_collect_window(spec, steps)
    assert released == [[], [], [], [10], [11, 12, 13]]
    assert [r[3] for r in acts[3] if r[2] == "E"] == [[10, 11, 12]]


# ---------------------------------------------------------------------------
# which collect_window calls carry a GPU plan
# ---------------------------------------------------------------------------


def _plan_of(into=list, ordered=True, windower=None, clock=None):
    import bytewax_b200.operators as op
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.operators import windowing as W
    from bytewax_b200.testing import TestingSource

    align = datetime(2022, 1, 1, tzinfo=timezone.utc)
    windower = windower or W.TumblingWindower(length=timedelta(seconds=10), align_to=align)
    clock = clock or W.EventClock(lambda v: align, wait_for_system_duration=timedelta(seconds=1))
    flow = Dataflow("plan")
    up = op.key_on("k", op.input("in", flow, TestingSource([])), lambda _v: "k")
    W.collect_window("collect", up, clock, windower, into=into, ordered=ordered)
    plans = []

    def walk(step):
        b = getattr(step, "builder", None)
        if b is not None and getattr(b, "_gpu_plan", None) is not None:
            plans.append(b._gpu_plan)
        for sub in getattr(step, "substeps", []) or []:
            walk(sub)

    for s in flow.substeps:
        walk(s)
    return plans[0] if plans else None


@pytest.mark.parametrize("into", [list, set, dict])
@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("shape", ["tumbling", "sliding"])
@pytest.mark.parametrize("clock", ["event", "system"])
def test_plan_carried(into, ordered, shape, clock):
    from bytewax_b200.operators import windowing as W

    align = datetime(2022, 1, 1, tzinfo=timezone.utc)
    w = (W.TumblingWindower(length=timedelta(seconds=10), align_to=align) if shape == "tumbling"
         else W.SlidingWindower(length=timedelta(seconds=60), offset=timedelta(seconds=7), align_to=align))
    c = W.SystemClock() if clock == "system" else W.EventClock(lambda v: align, wait_for_system_duration=timedelta.max)
    plan = _plan_of(into, ordered, w, c)
    assert isinstance(plan, W.GpuCollectWindowPlan)
    assert plan.into is into and plan.ordered is ordered and plan.windower is w and plan.clock is c and plan.step_id == "plan.collect"


def test_no_plan_off_the_device():
    from bytewax_b200.operators import windowing as W

    class MyList(list):
        pass

    align = datetime(2022, 1, 1, tzinfo=timezone.utc)
    assert _plan_of(MyList) is None
    assert _plan_of(windower=W.SessionWindower(gap=timedelta(seconds=5))) is None
    assert _plan_of(clock=W.EventClock(lambda v: align, timedelta(0), to_system_utc=lambda t: t)) is None
