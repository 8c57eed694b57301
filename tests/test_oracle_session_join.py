"""The session-join oracle (tests/session_join_oracle.py) against the reference's own session `join_window`
(tests/golden/session_join_cases.json, tools/gen_session_join_golden.py), its release rule, which calls carry a plan
for K10, and the host engine's merge rule.  CPU only."""

import json
import os
from datetime import datetime, timedelta, timezone

import pytest

from oracle.streams import rows_digest
from tests import session_join_oracle as sj

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "session_join_cases.json")))
CASES = GOLDEN["cases"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_case(name):
    c = CASES[name]
    stats = {}
    acts, _rel = sj.run_session_join(c["spec"], c["steps"], stats=stats)
    assert acts == c["acts"]
    # the reference reports merged ids (direct merges of the sessions that close); the oracle counts every merge
    assert stats["merges"] >= c["merges"] and (stats["merges"] > 0) == (c["merges"] > 0)


@pytest.mark.parametrize("seed", sj.SEEDED)
def test_oracle_matches_reference_seeded(seed):
    g = GOLDEN["seeded"][f"seed_{seed}"]
    spec, steps = sj.seeded_steps(seed, moving=seed % 3 != 0)
    acts, _rel = sj.run_session_join(spec, steps)
    assert [len(a) for a in acts] == g["rows"]
    assert rows_digest(acts) == g["sha256"]


def test_golden_covers_the_semantics():
    # each numbered item of the semantics the device restates has a named case; merge cases merge
    for name in ("merge_rule_first", "merge_rule_last", "merge_completes_under_survivor_id", "value_in_merged_away_session_last",
                 "first_by_id_not_nearest", "chained_merges_direct_ids", "three_way_merge_one_call"):
        assert CASES[name]["merges"] > 0, name
    for name in ("close_strict_boundary", "eof_near_utc_max", "never_discarded_keeps_watermark", "ordered_ties_stable",
                 "ordered_notify_wakes_queue_head", "gap_zero_same_ts_shares", "system_clock_moving_now"):
        assert name in CASES
    assert sum(c["spec"]["ordered"] is False for c in CASES.values()) >= 10
    assert {c["spec"]["sides"] for c in CASES.values()} >= {1, 2, 3, 4}
    assert len([n for n in CASES if n.startswith("ref_")]) == 5
    assert len(GOLDEN["seeded"]) >= 48 and sum(g["merges"] > 0 for g in GOLDEN["seeded"].values()) >= 4


def _all_cases():
    for name, c in CASES.items():
        yield name, c["spec"], c["steps"]
    for seed in sj.SEEDED:
        spec, steps = sj.seeded_steps(seed, moving=seed % 3 != 0)
        yield f"seed_{seed}", spec, steps


@pytest.mark.parametrize("name,spec,steps", list(_all_cases()), ids=lambda x: x if isinstance(x, str) else "")
def test_every_handle_released_once(name, spec, steps):
    """Each handle comes back exactly once by EOF, unless its session never closes (close >= UTC_MAX - gap)."""
    acts, rel = sj.run_session_join(spec, steps)
    flat = [h for r in rel for h in r]
    assert len(flat) == len(set(flat))
    given = {v for st in steps if st[0] == "batch" for v in st[5]}
    if name == "eof_near_utc_max":
        assert set(flat) < given
    else:
        assert set(flat) == given


@pytest.mark.parametrize("seed", [s for s in sj.SEEDED if sj.seeded_spec(s)["ordered"]])
def test_ordered_streams_never_merge(seed):
    stats = {}
    spec, steps = sj.seeded_steps(seed, moving=seed % 3 != 0)
    sj.run_session_join(spec, steps, stats=stats)
    assert stats["merges"] == 0


def test_which_calls_carry_a_plan():
    from bytewax_b200.operators import windowing as W

    clock = W.EventClock(lambda v: v, timedelta(0))
    sess = W.SessionWindower(timedelta(seconds=1))
    for ins in ("first", "last"):
        for n in (1, 2, 3, 4):
            p = W._join_window_plan(clock, sess, n, ins, "final", True)
            assert isinstance(p, W.GpuJoinWindowPlan) and p.windower is sess and p.sides == n
    assert W._join_window_plan(W.SystemClock(), sess, 2, "last", "running", False) is not None
    assert W._join_window_plan(clock, sess, 2, "product", "final", True) is None
    assert W._join_window_plan(clock, sess, 5, "last", "final", True) is None
    custom = W.EventClock(lambda v: v, timedelta(0), to_system_utc=lambda t: t)
    assert W._join_window_plan(custom, sess, 2, "last", "final", True) is None
    # collect_window over sessions stays on the host
    assert W._collect_window_plan("c", clock, sess, list, True) is None


def test_session_plans_route_to_the_session_join_step():
    from bytewax_b200 import engine
    from bytewax_b200.operators import windowing as W

    p = W._join_window_plan(W.EventClock(lambda v: v, timedelta(0)), W.SessionWindower(timedelta(seconds=1)), 2, "last", "final", True)
    st = engine._gpu_step_for("j", p)
    assert type(st) is engine._GpuSessionJoinWindowStep
    assert not isinstance(st, engine._GpuSessionStep)


EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)


def test_notify_case_pins_queue_head(monkeypatch):
    """`ordered_notify_wakes_queue_head` tells waking on queue[0]'s ts from waking on the smallest queued ts."""
    c = CASES["ordered_notify_wakes_queue_head"]

    def smallest(self):
        at = self.windower.notify_at()
        if self.ordered and self.queue:
            q = min(e[1] for e in self.queue)
            at = q if at is None else min(at, q)
        return at

    monkeypatch.setattr(sj.SessionJoinLogic, "notify_at", smallest)
    assert sj.run_session_join(c["spec"], c["steps"])[0] != c["acts"]


def _host_run(c):
    """The golden case through `run_main(gpu=False)`: one input per side, each fed as one batch.  The engine feeds the
    inputs' batches in input order, so the case's items must come in side order (checked here): then the host engine
    sees them in the case's order, and with the wait forever and no notify, batch boundaries change nothing."""
    import bytewax_b200.operators as op
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource, run_main

    spec, steps = c["spec"], c["steps"]
    assert all(st[0] == "batch" for st in steps) and spec["wait_us"] == sj.WAIT_FOREVER and not spec["ordered"]
    keys, ts, sides, vals = ([x for st in steps for x in st[i]] for i in (2, 3, 4, 5))
    assert sides == sorted(sides), "items must come in side order"
    down, meta = [], []
    flow = Dataflow("df")
    ins = [op.input(f"in{i}", flow, TestingSource([(str(k), (v, t)) for k, t, sd, v in zip(keys, ts, sides, vals) if sd == i], batch_size=1000))
           for i in range(spec["sides"])]
    clock = win.EventClock(lambda v: EPOCH + timedelta(microseconds=v[1]), timedelta.max,
                           now_getter=lambda: datetime(2030, 1, 1, tzinfo=timezone.utc))
    wo = win.join_window("j", clock, win.SessionWindower(timedelta(microseconds=spec["gap_us"])), *ins,
                         insert_mode=spec["insert_mode"], emit_mode=spec["emit_mode"], ordered=False)
    op.output("o", wo.down, TestingSink(down))
    op.output("m", wo.meta, TestingSink(meta))
    run_main(flow, gpu=False)
    us = lambda d: int((d - EPOCH) / timedelta(microseconds=1))  # noqa: E731
    e = [[int(k), w, "E", [None if v is None else v[0] for v in t]] for k, (w, t) in down]
    m = [[int(k), w, "M", [us(md.open_time), us(md.close_time), sorted(md.merged_ids)]] for k, (w, md) in meta]
    return e, m


@pytest.mark.parametrize("name", ["merge_rule_first", "merge_rule_last", "merge_rule_first_across_calls", "merge_rule_last_across_calls",
                                  "first_by_id_not_nearest", "value_in_merged_away_session_first"])
def test_host_engine_merge_rule(name):
    """The host engine's `_JoinWindowLogic.on_merge` is the reference's: "last" keeps the survivor's value."""
    c = CASES[name]
    e, m = _host_run(c)
    rows = [r for a in c["acts"] for r in a]
    assert e == [r for r in rows if r[2] == "E"]
    assert m == [r for r in rows if r[2] == "M"]
