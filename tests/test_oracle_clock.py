"""The moving-clock streams of tests/clock_streams.py reach the shapes they claim, on the oracle.  CPU only."""

import pytest

from tests import clock_streams as cs


@pytest.mark.parametrize("case", cs.all_cases(), ids=lambda c: c.name)
def test_builder_reaches_its_shapes(case):
    tr = cs.run(case)
    for i, want in case.claims.items():
        assert want <= tr.shapes[i], (case.name, i, sorted(want - tr.shapes[i]))
    # k_close_wake refuses exactly the notify phase the case names, and no other
    assert [i for i, r in enumerate(tr.refuse) if r] == ([] if case.refuse_at is None else [case.refuse_at])


@pytest.mark.parametrize("which", ["late_wake", "early_wake"])
def test_refused_notify_is_where_ordered_differs(which):
    """At the refused notify phase the ordered reference emits other rows than the same stream unordered -- what the
    device's due test computes -- so the refusal marks a real difference, not a guess."""
    case = cs.ordered_queue_head(which)
    ordered, unordered = cs.run(case), cs.run(case, ordered=False)
    i = case.refuse_at
    assert ordered.rows[i] != unordered.rows[i]
    assert ordered.rows[:i] == unordered.rows[:i]


def test_event_time_behind_the_clock_is_never_refused():
    """Ordered streams whose items never lead their arrival's system time (every 2026-clock and SystemClock-shaped
    stream): the ordered reference's notify phases emit exactly what the unordered ones do."""
    for case in (cs.wall_clock_2026(True), cs.ordered_queue_head("behind")):
        tr, un = cs.run(case), cs.run(case, ordered=False)
        assert not any(tr.refuse)
        assert [[r for r in a if r[2] != "M"] for a in tr.rows] == [[r for r in a if r[2] != "M"] for a in un.rows]


@pytest.mark.parametrize("n_keys,frac", [(100_000, 0.01), (100_000, 0.5), (100_000, 1.0)])
def test_many_keys_due_fraction(n_keys, frac):
    case = cs.many_keys(n_keys, frac, seed=int(frac * 100))
    tr = cs.run(case)
    assert abs(tr.due_frac[1] - frac) <= max(0.2 * frac, 0.002)
    assert sum(1 for r in tr.rows[1] if r[2] == "E") == round(tr.due_frac[1] * len(case.steps[0][2]))


def test_emit_capacity_rows():
    """emit_capacity's notify phase closes 128 windows, and nothing emits before it."""
    tr = cs.run(cs.emit_capacity())
    assert [sum(1 for r in a if r[2] == "E") for a in tr.rows] == [0, 128, 0]


def test_utc_min_floor_is_absolute():
    """A new key's watermark is UTC_MIN itself (windowing.py:245-248), not UTC_MIN + now: under a 2026 clock no row
    near UTC_MIN is late; the one late row is behind its own key's (ts - wait), near UTC_MAX."""
    tr = cs.run(cs.limits())
    late = [r for a in tr.rows for r in a if r[2] == "L"]
    assert [(k, p) for k, _w, _t, p in late] == [(5, 8)]


@pytest.mark.parametrize("windower", ["tumbling", "sliding"])
@pytest.mark.parametrize("reduction", ["count", "sum", "max", "min"])
def test_custom_to_system_utc_goes_to_the_host(windower, reduction):
    """The device's notify phase compares a window's close in event time with the system clock; the reference
    passes the close through `to_system_utc` first (windowing.py:1177-1178).  A custom one keeps the fold (count_window,
    reduce_window, max_window / min_window with the identity `by`) on the host; the default and a SystemClock reach
    the device."""
    from datetime import datetime, timedelta, timezone

    from bytewax_b200.operators import windowing as W

    align = datetime(2022, 1, 1, tzinfo=timezone.utc)
    win = (W.TumblingWindower(timedelta(seconds=10), align) if windower == "tumbling"
           else W.SlidingWindower(timedelta(seconds=10), timedelta(seconds=5), align))
    custom = W.EventClock(lambda v: v, timedelta(0), to_system_utc=lambda t: t + timedelta(hours=1))
    assert W._plan_for(reduction, custom, win, False) is None
    assert W._plan_for(reduction, W.EventClock(lambda v: v, timedelta(0)), win, False) is not None
    assert W._plan_for(reduction, W.SystemClock(), win, False) is not None


@pytest.mark.parametrize("seed", [1, 2])
def test_c1_reference_is_the_oracle(seed):
    """The vectorised reference of the C1-size stepping-clock case gives the oracle's rows, step for step, on the same
    stream at a small size (many late rows, keys discarded and back)."""
    case = cs.c1_stepping(4000, 500, 6, seed=seed, straggle=0.05)
    ref, tr = cs.c1_reference(case), cs.run(case)
    assert len(ref) == len(tr.rows)
    for (down, late), rows in zip(ref, tr.rows):
        assert down == [(k, w, p) for k, w, t, p in rows if t == "E"]
        assert [(k, w, i) for k, w, i, _t in late] == [(k, w, p) for k, w, t, p in rows if t == "L"]
    assert sum(len(d) for d, _ in ref) > 1000 and sum(len(l_) for _, l_ in ref) > 500


def test_many_keys_reference_is_the_oracle():
    case = cs.many_keys(20_000, 0.5, seed=3)
    ref, tr = cs.many_keys_reference(case), cs.run(case)
    for (down, late), rows in zip(ref, tr.rows):
        assert down == [(k, w, p) for k, w, t, p in rows if t == "E"] and not late
