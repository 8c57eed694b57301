"""Generate ``tests/golden/session_join_cases.json`` from the UNMODIFIED reference `join_window` over `SessionWindower`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_session_join_golden.py

Every case builds a real reference flow (``win.join_window`` over an ``EventClock`` and a ``SessionWindower``), pulls
the ``stateful_batch`` step's builder out of the step tree, and drives the reference's own ``_WindowLogic`` +
``_SessionWindowerLogic`` + ``_JoinWindowLogic`` with the engine rules of src/operators.rs:755-806 (ascending key string
per activation; a session logic never reports itself empty, so none is discarded), :808-858 (notify: every key whose
``notify_at()`` has come) and :862-894 (EOF).

Items are ``(key_str, (value, ts_us))`` on side ``side``; values are distinct ints, so they double as the handles the
device joins.  Hand-built cases store their rows in full, with the number of merges the reference made; every case
named for a merge is checked to merge.  The seeded streams of ``tests/session_join_oracle.py`` (``seeded_steps``)
store the SHA-256 of their rows.  The file holds data only.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import session_join_oracle as sj  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A = sj.S, sj.A
UTC_MAX = 253_402_300_799_999_999


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def join_builder(spec, now_getter):
    """The reference's `stateful_batch` builder of a session `join_window` flow; side values are ``(value, ts_us)``."""
    wait = timedelta.max if spec["wait_us"] == sj.WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda v: dt(v[1]), wait_for_system_duration=wait, now_getter=now_getter)
    windower = win.SessionWindower(gap=timedelta(microseconds=spec["gap_us"]))
    flow = Dataflow("g")
    sides = [op.input(f"in{i}", flow, TestingSource([])) for i in range(spec["sides"])]
    win.join_window("j", clock, windower, *sides, insert_mode=spec["insert_mode"], emit_mode=spec["emit_mode"],
                    ordered=spec["ordered"])
    return refstub.find_stateful_batch(flow).builder


def run_reference(spec, steps):
    """Rows per step (then EOF), and how many merges the reference's session windowers made."""
    now = [dt(steps[0][1])]
    builder = join_builder(spec, lambda: now[0])
    logics, acts = {}, []
    merges = [0]

    def conv(ks, events):
        rows = []
        for wid, tag, p in events:
            if tag == "E":
                rows.append([int(ks), wid, "E", [None if v is None else v[0] for v in p]])
            elif tag == "L":
                rows.append([int(ks), wid, "L", [p[0], p[1][0]]])
            else:
                rows.append([int(ks), wid, "M", [us(p.open_time), us(p.close_time), sorted(p.merged_ids)]])
        return rows

    def done_with(ks, res, rows):
        events, done = res
        assert not done  # session state is never discarded (windowing.py:798-806)
        rows.extend(conv(ks, list(events)))

    for step in steps:
        now[0] = dt(step[1])
        rows = []
        if step[0] == "batch":
            grouped = {}
            for k, t, sd, v in zip(step[2], step[3], step[4], step[5]):
                grouped.setdefault(str(k), []).append((sd, (v, t)))
            for ks in sorted(grouped):
                logic = logics.get(ks)
                if logic is None:
                    logic = logics[ks] = builder(None)
                done_with(ks, logic.on_batch(grouped[ks]), rows)
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now[0]:
                    done_with(ks, logics[ks].on_notify(), rows)
        acts.append(rows)
    rows = []
    for ks in sorted(logics):
        done_with(ks, logics[ks].on_eof(), rows)
    acts.append(rows)
    merges[0] = sum(len(r[3][2]) for act in acts for r in act if r[2] == "M")
    return acts, merges[0]


def spec_(ins="last", emit="final", ordered=True, sides=2, gap=10 * S, wait=0):
    return dict(insert_mode=ins, emit_mode=emit, ordered=ordered, sides=sides, gap_us=gap, wait_us=wait)


class Steps:
    """Builds golden steps; every value is a fresh int (its handle)."""

    def __init__(self, now=A + 10**6 * S):
        self.steps, self.n, self.now = [], 0, now

    def batch(self, *items, now=None):
        """``items``: ``(key, ts, side)``."""
        if now is not None:
            self.now = now
        k, t, s = ([it[i] for it in items] for i in range(3))
        self.steps.append(["batch", self.now, k, t, s, list(range(self.n, self.n + len(items)))])
        self.n += len(items)
        return self

    def notify(self, now):
        self.now = now
        self.steps.append(["notify", now])
        return self


def main():
    cases = {}

    def add(name, spec, st, check=None, cite=None, merges=False):
        acts, n_merges = run_reference(spec, st.steps)
        if check is not None:
            assert check(acts), (name, acts)
        assert (n_merges > 0) == merges, (name, n_merges)  # a case named for a merge must merge; the others must not
        cases[name] = dict(spec=spec, steps=st.steps, acts=acts, cite=cite, merges=n_merges)

    def tags(acts, tag):
        return [r for act in acts for r in act if r[2] == tag]

    F = sj.WAIT_FOREVER
    # --- the reference's own session joins: pytests/operators/windowing/test_join_window.py (gap 10 s, wait forever,
    # one key, the left input before the right); values 1.. are the handles 0..
    T0 = us(datetime(2024, 1, 1, tzinfo=timezone.utc))
    ref = "pytests/operators/windowing/test_join_window.py"
    add("ref_first_complete", spec_("first", "complete", wait=F),
        Steps().batch((0, T0, 0), (0, T0 + 2 * S, 1), (0, T0 + S, 1)), check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2]],
        cite=ref + ":71-86")
    add("ref_last_complete", spec_("last", "complete", wait=F),
        Steps().batch((0, T0, 0), (0, T0 + S, 1)), check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 1]], cite=ref + ":89-103")
    add("ref_last_final", spec_("last", "final", wait=F),
        Steps().batch((0, T0, 0), (0, T0 + S, 1), (0, T0 + 2 * S, 1)), check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2]],
        cite=ref + ":106-121")
    add("ref_default_last_final", spec_(wait=F),
        Steps().batch((0, T0, 0), (0, T0 + S, 1), (0, T0 + 2 * S, 1)), check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2]],
        cite=ref + ":124-139")
    add("ref_last_running", spec_("last", "running", wait=F),
        Steps().batch((0, T0, 0), (0, T0 + S, 1), (0, T0 + 2 * S, 1)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, None], [0, 1], [0, 2]], cite=ref + ":142-159")

    # --- 1. the merge rule: session 0 holds {0: h0, 1: h2}, session 1 {0: h1}; h3 (side 1) at A+10 extends session 0,
    # which then absorbs session 1.  first: h3 is dropped, h1 wins side 0 -> (h1, h2); last: h3 replaces h2 and the
    # survivor keeps h0 -> (h0, h3).  (Items in side order, as the host-engine check feeds them.)
    merge = Steps().batch((1, A, 0), (1, A + 20 * S, 0), (1, A, 1), (1, A + 10 * S, 1))
    add("merge_rule_first", spec_("first", "final", ordered=False, wait=F), merge,
        check=lambda a: [r[3] for r in tags(a, "E")] == [[1, 2]], merges=True)
    add("merge_rule_last", spec_("last", "final", ordered=False, wait=F), merge,
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 3]], merges=True)
    # the issue's shape across two activations: survivor {0: a, 1: c} absorbs {0: b}; last keeps a, first takes b
    two = Steps().batch((2, A, 0), (2, A + 20 * S, 0)).batch((2, A + S, 1), (2, A + 10 * S, 1))
    add("merge_rule_last_across_calls", spec_("last", "final", ordered=False, wait=F), two, merges=True)
    add("merge_rule_first_across_calls", spec_("first", "final", ordered=False, wait=F), two, merges=True)
    # the merge completes the tuple: complete emits under the survivor's id (0) and clears; running emits
    comp = Steps().batch((3, A, 0), (3, A + 20 * S, 1), (3, A + 10 * S, 0))
    add("merge_completes_under_survivor_id", spec_("first", "complete", ordered=False, wait=F), comp,
        check=lambda a: [[r[1], r[3]] for r in tags(a, "E")] == [[0, [0, 1]]], merges=True)
    add("merge_running_emits", spec_("last", "running", ordered=False, wait=F), comp, merges=True)
    # --- 2. a value whose own extension merged its session away: it goes to session 0, which merges into 1 afterwards
    add("value_in_merged_away_session_last", spec_("last", "final", ordered=False, wait=F),
        Steps().batch((4, A + 20 * S, 0), (4, A, 1), (4, A + 10 * S, 0)),
        check=lambda a: [[r[1], r[3]] for r in tags(a, "E")] == [[1, [2, 1]]], merges=True)
    add("value_in_merged_away_session_first", spec_("first", "complete", ordered=False, sides=3, wait=F),
        Steps().batch((4, A + 20 * S, 0), (4, A, 1), (4, A + 10 * S, 2)), merges=True)
    # --- 3. which session takes a value: A+13 is 7 s before session 0 and 5 s after session 1; the first by id (0)
    # takes it, not the nearest (1), and the survivor 1 keeps its own side 0 under last -> (h1)
    add("first_by_id_not_nearest", spec_("last", "final", ordered=False, sides=1, wait=F),
        Steps().batch((5, A + 20 * S, 0), (5, A + 8 * S, 0), (5, A + 13 * S, 0)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[1]], merges=True)
    # --- 4. chained merges: 1 absorbs 2 in one call, 0 absorbs 1 in the next; merged ids are direct merges only
    add("chained_merges_direct_ids", spec_("last", "final", ordered=False, sides=2, gap=10 * S, wait=F),
        Steps().batch((6, A, 0), (6, A + 15 * S, 1), (6, A + 30 * S, 0), (6, A + 22 * S, 1)).batch((6, A + 7 * S, 1)),
        check=lambda a: [r[3] for r in tags(a, "M")] == [[A, A + 30 * S, [1]]], merges=True)
    add("three_way_merge_one_call", spec_("first", "running", ordered=False, sides=3, gap=6 * S, wait=F),
        Steps().batch((7, A, 0), (7, A + 12 * S, 1), (7, A + 24 * S, 2), (7, A + 6 * S, 1), (7, A + 18 * S, 0)),
        check=lambda a: [r[3][2] for r in tags(a, "M")] == [[1, 2]], merges=True)
    # --- 5. close and EOF boundaries: close_after = watermark - gap; A+3 s with wait 1 s, gap 2 s puts it exactly at
    # session 0's close (stays open), A+3 s + 1 us one past (closes)
    add("close_strict_boundary", spec_("last", "final", ordered=False, gap=2 * S, wait=S),
        Steps().batch((8, A, 0)).batch((8, A + 3 * S, 1)).batch((8, A + 3 * S + 1, 0)),
        check=lambda a: not tags(a[:2], "M") and [r[1] for r in tags(a[2:3], "M")] == [0])
    add("eof_near_utc_max", spec_("last", "final", ordered=True, gap=2 * S, wait=0),
        Steps().batch((9, UTC_MAX - S, 0), (10, UTC_MAX - 3 * S, 1), (11, UTC_MAX - 2 * S, 0)),
        check=lambda a: [r[0] for r in tags(a, "M")] == [10])
    # --- 6. never discarded: key 12's only session closes at a notify; its clock stays (and drifts with `now`), so A+5
    # and A+40 are late (under K8's discard the first would open a new window)
    add("never_discarded_keeps_watermark", spec_("last", "final", ordered=False, gap=S, wait=0),
        Steps(now=A).batch((12, A + 20 * S, 0), now=A).notify(A + 21 * S).batch((12, A + 5 * S, 1), now=A + 22 * S)
        .batch((12, A + 40 * S, 1)),
        check=lambda a: len(tags(a, "L")) == 2 and [r[1] for r in tags(a, "M")] == [0])
    # --- 7. ordered mode never merges: ties in arrival order, a queue across activations, the notify waking on queue[0]
    add("ordered_ties_stable", spec_("last", "running", ordered=True, sides=2, gap=S, wait=5 * S),
        Steps().batch((1, A + 3 * S, 0), (1, A + S, 1), (1, A + S, 0), (1, A + 3 * S, 1), (1, A + S, 0), (1, A + 9 * S, 0))
        .batch((1, A + 30 * S, 1)))
    add("ordered_queue_across_activations", spec_("first", "complete", ordered=True, sides=2, gap=2 * S, wait=4 * S),
        Steps().batch((1, A + 6 * S, 0), (1, A + 2 * S, 1)).batch((1, A + 7 * S, 1), (1, A + 3 * S, 0))
        .batch((1, A + 9 * S, 0)).batch((1, A + 15 * S, 1), (2, A, 0)))
    # queue[0] (ts A+8) is not the smallest queued ts (A+5): the notify wakes at A+8 once `now` drifts the watermark
    # (running, and a notify at A+6, between the smallest queued ts and queue[0]'s: waking on the smallest ts would emit
    # rows there instead of at A+8)
    add("ordered_notify_wakes_queue_head", spec_("last", "running", ordered=True, sides=2, gap=20 * S, wait=10 * S),
        Steps(now=A).batch((4, A + 8 * S, 0), (4, A + 5 * S, 1), (4, A + 12 * S, 1), now=A)
        .notify(A + 4 * S).notify(A + 6 * S).notify(A + 8 * S).notify(A + 9 * S).notify(A + 60 * S),
        check=lambda a: not a[2] and a[3])
    add("wait_forever_flush_at_eof", spec_("last", "final", ordered=True, sides=3, gap=S, wait=F),
        Steps().batch((1, A + 9 * S, 2), (1, A + 1 * S, 0), (1, A + 5 * S, 1)).batch((1, A, 1), (2, A + 3 * S, 0), (1, A + 2 * S, 2)),
        check=lambda a: not any(a[:-1]) and len(tags(a, "M")) == 4)
    # --- side counts, gap 0 ------------------------------------------------------------------------------------------------
    add("one_side", spec_("first", "complete", ordered=False, sides=1, gap=S, wait=S),
        Steps().batch((1, A, 0), (1, A + 1, 0), (2, A + S, 0)).batch((1, A + 10 * S, 0)))
    add("four_sides_partial", spec_("last", "final", ordered=True, sides=4, gap=S, wait=S),
        Steps().batch((1, A, 3), (1, A + S, 1), (2, A, 0), (2, A + 1, 2), (2, A + 2, 3), (2, A + 3, 1)).batch((1, A + 50 * S, 0)))
    add("gap_zero_same_ts_shares", spec_("last", "running", ordered=False, sides=2, gap=0, wait=0),
        Steps().batch((1, A, 0), (1, A, 1), (1, A + 1, 0)).batch((1, A + 1, 1), (1, A + 5, 0)),
        check=lambda a: len(tags(a, "M")) == 3)
    # --- clocks -----------------------------------------------------------------------------------------------------------
    # SystemClock: every item is stamped with the batch's system time and the wait is 0
    sc = Steps(now=A)
    for i, k in enumerate((1, 2, 1, 1, 2, 1)):
        now = A + i * 3 * S
        sc.batch((k, now, i % 2), (k, now, (i + 1) % 2), now=now)
        if i % 2:
            sc.notify(now + 2 * S)
    add("system_clock_moving_now", spec_("last", "running", ordered=True, sides=2, gap=2 * S, wait=0), sc.notify(A + 60 * S))
    add("moving_clock_drift_late", spec_("first", "complete", ordered=False, sides=2, gap=S, wait=2 * S),
        Steps(now=A + S).batch((7, A + S, 0), (8, A + S, 1), now=A + S).batch((7, A + 2 * S, 1), now=A + 21 * S)
        .batch((8, A + 25 * S, 0), now=A + 22 * S).notify(A + 40 * S))
    # --- keys whose decimal text orders differently from their value -------------------------------------------------------
    keys = [0, 2**64 - 1, 2**63] + [10**k - 1 for k in range(1, 20)] + [10**k for k in range(1, 20)]
    add("digit_boundary_keys", spec_("last", "running", ordered=False, sides=2, gap=S, wait=0),
        Steps().batch(*[(k, A + (i % 3) * S, i % 2) for i, k in enumerate(keys)]).batch(*[(k, A + 5 * S, 1) for k in keys[::-1]]))

    seeded = {}
    for seed in sj.SEEDED:
        spec, steps = sj.seeded_steps(seed, moving=seed % 3 != 0)
        acts, n_merges = run_reference(spec, steps)
        assert not (spec["ordered"] and n_merges), seed  # ordered mode never merges
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts], merges=n_merges)
    path = os.path.join(ROOT, "tests", "golden", "session_join_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
