"""The session product-join oracle (tests/session_product_join_oracle.py) against the reference's own
`join_window(insert_mode="product")` over `SessionWindower` (tests/golden/session_product_join_cases.json,
tools/gen_session_product_join_golden.py), its release rule, which calls carry a plan for K16, and the step the engine
builds for it.  CPU only."""

import json
import os
from datetime import timedelta

import pytest

from oracle.streams import rows_digest
from tests import session_product_join_oracle as sp

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "session_product_join_cases.json")))
CASES = GOLDEN["cases"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_case(name):
    c = CASES[name]
    stats = {}
    acts, _rel = sp.run_session_product_join(c["spec"], c["steps"], stats=stats)
    assert acts == c["acts"]
    assert stats["merges"] == c["merges"]


@pytest.mark.parametrize("seed", sp.SEEDED)
def test_oracle_matches_reference_seeded(seed):
    g = GOLDEN["seeded"][f"seed_{seed}"]
    spec, steps = sp.seeded_steps(seed, moving=seed % 3 != 0)
    stats = {}
    acts, _rel = sp.run_session_product_join(spec, steps, stats=stats)
    assert [len(a) for a in acts] == g["rows"]
    assert rows_digest(acts) == g["sha256"]
    assert stats["merges"] == g["merges"]


def test_golden_covers_the_semantics():
    for name in ("survivor_values_after_merge_found_final", "survivor_values_after_merge_found_running", "complete_clear_before_merge",
                 "merge_completes", "running_staged_twice", "value_in_merged_away_session", "final_merged_closed_by_notify"):
        assert CASES[name]["merges"] > 0, name
    for name in ("chain_running", "chain_complete_emits_at_last_merge", "chain_complete_clears_midway", "chain_final_merged_ids"):
        assert CASES[name]["chains"] > 0, name
    for name in ("late_items", "ordered_ties_running", "ordered_queue_complete", "stepping_clock_notify_running", "eof_closes_open_sessions"):
        assert name in CASES
    assert {(c["spec"]["emit_mode"], c["spec"]["sides"]) for c in CASES.values()} >= {(e, n) for e in sp.EMITS for n in (1, 2, 3, 4)}
    assert any(None in r[3] for c in CASES.values() for a in c["acts"] for r in a if r[2] == "E")
    assert any(r[2] == "L" for c in CASES.values() for a in c["acts"] for r in a)
    assert len(GOLDEN["seeded"]) >= 48 and sum(g["merges"] > 0 for g in GOLDEN["seeded"].values()) >= 4


def _all_cases():
    for name, c in CASES.items():
        yield name, c["spec"], c["steps"]
    for seed in sp.SEEDED:
        spec, steps = sp.seeded_steps(seed, moving=seed % 3 != 0)
        yield f"seed_{seed}", spec, steps


@pytest.mark.parametrize("name,spec,steps", list(_all_cases()), ids=lambda x: x if isinstance(x, str) else "")
def test_every_handle_released_once(name, spec, steps):
    """Each handle comes back exactly once by EOF."""
    _acts, rel = sp.run_session_product_join(spec, steps)
    flat = [h for r in rel for h in r]
    assert len(flat) == len(set(flat))
    assert set(flat) == {v for st in steps if st[0] == "batch" for v in st[5]}


@pytest.mark.parametrize("seed", [s for s in sp.SEEDED if sp.seeded_spec(s)["ordered"]])
def test_ordered_streams_never_merge(seed):
    stats = {}
    spec, steps = sp.seeded_steps(seed, moving=seed % 3 != 0)
    sp.run_session_product_join(spec, steps, stats=stats)
    assert stats["merges"] == 0


def test_which_calls_carry_a_plan():
    from bytewax_b200.operators import windowing as W

    clock = W.EventClock(lambda v: v, timedelta(0))
    sess = W.SessionWindower(timedelta(seconds=1))
    for n in (1, 2, 3, 4):
        p = W._session_product_join_window_plan(clock, sess, n, "product", "final", True)
        assert isinstance(p, W.GpuJoinWindowPlan) and p.windower is sess and p.sides == n and p.insert_mode == "product"
    assert W._session_product_join_window_plan(W.SystemClock(), sess, 2, "product", "running", False) is not None
    assert W._session_product_join_window_plan(clock, sess, 5, "product", "final", True) is None
    custom = W.EventClock(lambda v: v, timedelta(0), to_system_utc=lambda t: t)
    assert W._session_product_join_window_plan(custom, sess, 2, "product", "final", True) is None
    # only product over sessions: K8, K10 and K14 keep theirs, and `_join_window_plan` still has none for this
    assert W._session_product_join_window_plan(clock, sess, 2, "last", "final", True) is None
    assert W._session_product_join_window_plan(clock, W.TumblingWindower(timedelta(seconds=1), W.UTC_MIN), 2, "product", "final", True) is None
    assert W._join_window_plan(clock, sess, 2, "product", "final", True) is None


def test_join_window_attaches_the_plan():
    from bytewax_b200 import operators as op
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.operators import windowing as W
    from bytewax_b200.testing import TestingSource

    flow = Dataflow("df")
    sides = [op.input(f"in{i}", flow, TestingSource([])) for i in range(3)]
    W.join_window("j", W.EventClock(lambda v: v, timedelta(0)), W.SessionWindower(timedelta(seconds=1)), *sides, insert_mode="product")
    plans = [getattr(s, "_gpu_plan", None) for s in _walk(flow)]
    p = [x for x in plans if x is not None]
    assert len(p) == 1 and p[0].insert_mode == "product" and p[0].sides == 3 and isinstance(p[0].windower, W.SessionWindower)


def _walk(flow):
    stack = list(flow.substeps)
    while stack:
        s = stack.pop()
        yield s
        stack.extend(getattr(s, "substeps", []))


def test_session_product_plans_route_to_their_step():
    from bytewax_b200 import engine
    from bytewax_b200.operators import windowing as W

    p = W._session_product_join_window_plan(W.EventClock(lambda v: v, timedelta(0)), W.SessionWindower(timedelta(seconds=1)), 2, "product",
                                            "final", True)
    st = engine._gpu_step_for("j", p)
    assert type(st) is engine._GpuSessionProductJoinWindowStep
    assert st.gap_us == 1_000_000
    # the product step over tumbling windows and the first / last session step are unchanged
    q = W._join_window_plan(W.EventClock(lambda v: v, timedelta(0)), W.TumblingWindower(timedelta(seconds=1), W.UTC_MIN), 2, "product",
                            "final", True)
    assert type(engine._gpu_step_for("j", q)) is engine._GpuProductJoinWindowStep
    r = W._join_window_plan(W.EventClock(lambda v: v, timedelta(0)), W.SessionWindower(timedelta(seconds=1)), 2, "last", "final", True)
    assert type(engine._gpu_step_for("j", r)) is engine._GpuSessionJoinWindowStep
