"""The `join_window(insert_mode="product")` restatement (tests/product_join_window_oracle.py) against rows of the
reference's own, unmodified `_WindowLogic` + `_SlidingWindowerLogic` + `_JoinWindowLogic`
(tests/golden/product_join_window_cases.json, made by tools/gen_product_join_window_golden.py); which `join_window`
calls carry a device plan; and the host engine's rows for the reference guide's product example."""

import json
import os
from datetime import datetime, timedelta, timezone

import pytest

import bytewax_b200.operators as op
import bytewax_b200.operators.windowing as win
from bytewax_b200.dataflow import Dataflow
from bytewax_b200.testing import TestingSink, TestingSource, run_main
from oracle.streams import rows_digest
from tests import product_join_window_oracle as po

S, A = po.S, po.A
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "product_join_window_cases.json")

with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_case_list(golden):
    want = {"guide_bee_product", "final_side_empty_at_close", "one_side", "four_sides_with_gaps", "complete_refills_and_reemits",
            "complete_nothing_at_close_after_clear", "running_empty_sides", "sliding_clear_while_lower_window_holds",
            "late_sliding_all_windows", "ordered_out_of_order_ts", "moving_clock_notifies", "wait_forever_flush_at_eof",
            "near_utc_max"}
    assert want <= set(golden["cases"])
    assert len(golden["seeded"]) >= 40
    assert {c["spec"]["emit_mode"] for c in golden["cases"].values()} == {"complete", "final", "running"}


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hand_built_case(golden, name):
    case = golden["cases"][name]
    acts, released = po.run_product_join_window(case["spec"], case["steps"])
    assert acts == case["acts"]
    # every handle is released exactly once
    vals = [v for st in case["steps"] if st[0] == "batch" for v in st[5]]
    assert sorted(h for r in released for h in r) == sorted(vals)


def test_seeded_streams(golden):
    for seed in po.SEEDED:
        spec, steps = po.seeded_steps(seed, moving=seed % 3 != 0)
        acts, released = po.run_product_join_window(spec, steps)
        want = golden["seeded"][f"seed_{seed}"]
        assert [len(a) for a in acts] == want["rows"], seed
        assert rows_digest(acts) == want["sha256"], seed
        vals = [v for st in steps if st[0] == "batch" for v in st[5]]
        assert sorted(h for r in released for h in r) == sorted(vals)


def test_clear_while_a_lower_window_holds_the_value(golden):
    """In `complete` mode a sliding window can clear a value that a lower window still holds: window 1 clears value 0 in
    the second call while window 0 keeps it; the value is released only in the third, when window 0 clears it too."""
    case = golden["cases"]["sliding_clear_while_lower_window_holds"]
    acts, released = po.run_product_join_window(case["spec"], case["steps"])
    assert [r[1] for r in acts[1]] == [1] and [r[1] for r in acts[2]] == [0]
    assert 0 not in released[1] and 0 in released[2]


FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)


def _plan(insert_mode="product", windower=None, sides=2, **clock_kw):
    clock = win.EventClock(lambda v: v, timedelta(seconds=1), now_getter=lambda: FROZEN, **clock_kw)
    windower = windower or win.TumblingWindower(timedelta(seconds=1), FROZEN)
    return win._join_window_plan(clock, windower, sides, insert_mode, "final", True)


def test_which_calls_carry_a_product_plan():
    for sides in (1, 2, 3, 4):
        p = _plan(sides=sides)
        assert p is not None and p.insert_mode == "product" and p.sides == sides
    assert _plan(windower=win.SlidingWindower(timedelta(seconds=3), timedelta(seconds=1), FROZEN)).insert_mode == "product"
    assert win._join_window_plan(win.SystemClock(), win.TumblingWindower(timedelta(seconds=1), FROZEN), 2, "product", "running", False)
    assert _plan(windower=win.SessionWindower(timedelta(seconds=1))) is None
    assert _plan(sides=5) is None
    assert _plan(to_system_utc=lambda t: t) is None
    assert _plan("last", windower=win.SessionWindower(timedelta(seconds=1))) is not None


def test_host_engine_guide_example():
    """docs/guide/concepts/joins.md:641-728: Bee's name joined with both of her emails in one hour window."""
    at = datetime(2023, 12, 14, tzinfo=timezone.utc)
    names = [("123", {"at": at, "name": "Bee"})]
    emails = [("123", {"at": at + timedelta(minutes=15), "email": "bee@bytewax.io"}),
              ("123", {"at": at + timedelta(minutes=30), "email": "bee@example.com"})]
    down = []
    flow = Dataflow("df")
    sides = [op.input(f"in{i}", flow, TestingSource(items)) for i, items in enumerate((names, emails))]
    clock = win.EventClock(ts_getter=lambda x: x["at"], wait_for_system_duration=timedelta(0), now_getter=lambda: FROZEN)
    windower = win.TumblingWindower(length=timedelta(hours=1), align_to=datetime(2023, 1, 1, tzinfo=timezone.utc))
    wo = win.join_window("join", clock, windower, *sides, insert_mode="product")
    op.output("out", wo.down, TestingSink(down))
    run_main(flow)
    assert [(k, w, tuple(v["name"] if "name" in v else v["email"] for v in t)) for k, (w, t) in down] == [
        ("123", 8328, ("Bee", "bee@bytewax.io")), ("123", 8328, ("Bee", "bee@example.com"))]
