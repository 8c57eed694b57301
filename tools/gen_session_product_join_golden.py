"""Generate ``tests/golden/session_product_join_cases.json`` from the UNMODIFIED reference
`join_window(insert_mode="product")` over `SessionWindower`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_session_product_join_golden.py

Every case builds a real reference flow (``win.join_window`` over an ``EventClock`` and a ``SessionWindower``), pulls the
``stateful_batch`` step's builder out of the step tree, and drives the reference's own ``_WindowLogic`` +
``_SessionWindowerLogic`` + ``_JoinWindowLogic`` with the engine rules of src/operators.rs:755-806 (ascending key string
per activation; a session logic never reports itself empty), :808-858 (notify) and :862-894 (EOF), as
``tools/gen_session_join_golden.py`` does.

Items are ``(key_str, (value, ts_us))`` on side ``side``; values are distinct ints, so they double as the handles the
device joins.  Hand-built cases store their rows in full, with the number of merges the reference made and the number of
calls in which one key's merge queue CHAINED (a session took another in and was then merged away itself); every case
named for a merge is checked to merge, every case named for a chain to chain.  The seeded streams of
``tests/session_product_join_oracle.py`` store the SHA-256 of their rows.  The file holds data only.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import session_product_join_oracle as sp  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A = sp.S, sp.A
F = sp.WAIT_FOREVER


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def join_builder(spec, now_getter):
    """The reference's `stateful_batch` builder of a session product `join_window` flow; side values are ``(value, ts_us)``."""
    wait = timedelta.max if spec["wait_us"] == F else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda v: dt(v[1]), wait_for_system_duration=wait, now_getter=now_getter)
    windower = win.SessionWindower(gap=timedelta(microseconds=spec["gap_us"]))
    flow = Dataflow("g")
    sides = [op.input(f"in{i}", flow, TestingSource([])) for i in range(spec["sides"])]
    win.join_window("j", clock, windower, *sides, insert_mode="product", emit_mode=spec["emit_mode"], ordered=spec["ordered"])
    return refstub.find_stateful_batch(flow).builder


def run_reference(spec, steps):
    """Rows per step (then EOF), the merges the reference's session windowers made, and the calls whose merge queue
    chained."""
    now = [dt(steps[0][1])]
    builder = join_builder(spec, lambda: now[0])
    logics, acts = {}, []
    stats = dict(merges=0, chains=0)

    def watch(logic):
        # the windower's merge queue of each call, as `_handle_merged` takes it
        wdr = logic.windower
        merged = wdr.merged

        def take():
            q = list(merged())
            stats["merges"] += len(q)
            if any(t == o2 for i, (_, t) in enumerate(q) for o2, _ in q[i + 1:]):
                stats["chains"] += 1
            return q

        wdr.merged = take
        return logic

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
                    logic = logics[ks] = watch(builder(None))
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
    return acts, stats


def spec_(emit="final", ordered=False, sides=2, gap=10 * S, wait=F):
    return dict(emit_mode=emit, ordered=ordered, sides=sides, gap_us=gap, wait_us=wait)


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

    def add(name, spec, st, check=None, merges=False, chains=False):
        acts, stats = run_reference(spec, st.steps)
        if check is not None:
            assert check(acts), (name, acts)
        # a case named for a merge (a chain) must merge (chain); the others must not
        assert (stats["merges"] > 0) == merges, (name, stats)
        assert (stats["chains"] > 0) == chains, (name, stats)
        cases[name] = dict(spec=spec, steps=st.steps, acts=acts, merges=stats["merges"], chains=stats["chains"])

    def tags(acts, tag):
        return [r for act in acts for r in act if r[2] == tag]

    # --- every emit mode x 1 to 4 sides, no merge: key 1 fills sides 0 and the last one, key 2 only side 0, so empty
    # sides give None; a second call adds to both
    for emit in sp.EMITS:
        for n in range(1, 5):
            add(f"modes_{emit}_{n}_sides", spec_(emit, sides=n, gap=S, wait=S),
                Steps().batch((1, A, 0), (2, A, 0), (1, A + 1, n - 1), (1, A + 2, 0), (2, A + 3, 0))
                .batch((1, A + 4, n - 1), (2, A + 5, 0), (1, A + 6, n // 2)).batch((3, A + 20 * S, 0)),
                check=lambda a, n=n, emit=emit: n == 1 or emit == "complete" or any(None in r[3] for r in tags(a, "E")))
    # --- survivor values played after their merge was found precede the merged-away list: sessions 0 {s0: 0} and
    # 1 {s1: 1}; A+10 (side 1) extends 0 and finds 1 -> 0; A+5 (side 0) and A+12 (side 1) land in 0 before the merge
    surv = Steps().batch((1, A, 0), (1, A + 20 * S, 1)).batch((1, A + 10 * S, 1), (1, A + 5 * S, 0), (1, A + 12 * S, 1))
    add("survivor_values_after_merge_found_final", spec_("final"), surv,
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2], [0, 4], [0, 1], [3, 2], [3, 4], [3, 1]], merges=True)
    add("survivor_values_after_merge_found_running", spec_("running"), surv, merges=True)
    # --- a merge chain within one call: X (A), Y (A+20), Z (A+40), gap 10; A+30 bridges Y and Z, queueing Z -> Y; A+10
    # bridges X and Y, queueing Y -> X; the queue gives Y = Y + Z, then X = X + (Y + Z)
    add("chain_running", spec_("running"),
        Steps().batch((1, A, 0), (1, A + 20 * S, 1), (1, A + 40 * S, 0), (1, A + 40 * S + 1, 1))
        .batch((1, A + 30 * S, 0), (1, A + 10 * S, 1)), merges=True, chains=True)
    # complete: X {s0}, Y {s1}, Z {s2}; nothing is complete until (Y + Z) joins X: one emission of 2 x 2 x 1
    add("chain_complete_emits_at_last_merge", spec_("complete", sides=3),
        Steps().batch((1, A, 0), (1, A + 20 * S, 1), (1, A + 40 * S, 2))
        .batch((1, A + 30 * S, 1), (1, A + 10 * S, 0)),
        check=lambda a: len(tags(a[1:2], "E")) == 4, merges=True, chains=True)
    # complete: Z -> Y completes Y and clears it, so Y -> X moves nothing; a later value completes X alone
    add("chain_complete_clears_midway", spec_("complete", sides=2),
        Steps().batch((1, A, 0), (1, A + 20 * S, 0), (1, A + 40 * S, 1))
        .batch((1, A + 30 * S, 0), (1, A + 10 * S, 0)).batch((1, A + 2 * S, 1)),
        check=lambda a: len(tags(a[1:2], "E")) == 2 and len(tags(a[2:3], "E")) == 2, merges=True, chains=True)
    add("chain_final_merged_ids", spec_("final", sides=2),
        Steps().batch((1, A, 0), (1, A + 20 * S, 1), (1, A + 40 * S, 0), (2, A, 1))
        .batch((1, A + 30 * S, 1), (1, A + 10 * S, 0), (2, A + S, 0)),
        check=lambda a: [r[3][2] for r in tags(a, "M") if r[0] == 1] == [[1]], merges=True, chains=True)
    # --- a "complete" clear in the merged-away session earlier in the same call: only its current generation moves
    add("complete_clear_before_merge", spec_("complete"),
        Steps().batch((1, A, 0), (1, A + 20 * S, 0))
        .batch((1, A + 20 * S + 1, 1), (1, A + 21 * S, 0), (1, A + 10 * S, 0)).batch((1, A + 5 * S, 1)),
        check=lambda a: [r[3] for r in tags(a[2:3], "E")] == [[0, 5], [4, 5], [3, 5]], merges=True)
    # --- the merge itself completes: the survivor holds only side 0, the merged-away session only side 1
    add("merge_completes", spec_("complete"),
        Steps().batch((1, A, 0), (1, A + 20 * S, 1)).batch((1, A + 10 * S, 0)).batch((1, A + 11 * S, 1)),
        check=lambda a: [[r[1], r[3]] for r in tags(a[1:2], "E")] == [[0, [0, 1]], [0, [2, 1]]] and not tags(a[2:], "E"),
        merges=True)
    # --- running: B emits before the merge, A after it: B's value is staged under B's and A's coordinates in one call
    add("running_staged_twice", spec_("running"),
        Steps().batch((1, A, 0), (1, A + 20 * S, 1)).batch((1, A + 21 * S, 0), (1, A + 10 * S, 1)), merges=True)
    # --- a value whose own extension merged its session away goes to that session, which merges afterwards
    add("value_in_merged_away_session", spec_("running", sides=3),
        Steps().batch((4, A + 20 * S, 0), (4, A, 1), (4, A + 10 * S, 2)), merges=True)
    # --- final over merged sessions closed by the clock, with the meta rows' merged ids
    add("final_merged_closed_by_notify", spec_("final", sides=2, gap=2 * S, wait=10 * S),
        Steps(now=A).batch((1, A, 0), (1, A + 4 * S, 1), (2, A, 1), now=A).batch((1, A + 2 * S, 0), (1, A + 3 * S, 1), now=A + S)
        .notify(A + 5 * S).notify(A + 20 * S),
        check=lambda a: [r[3][2] for r in tags(a, "M") if r[0] == 1] == [[1]], merges=True)
    # --- late items: one row each, window -1, and their handles go at once
    add("late_items", spec_("final", sides=2, gap=S, wait=S),
        Steps().batch((1, A + 10 * S, 0), (2, A + 10 * S, 1)).batch((1, A, 1), (1, A + 10 * S, 1), (2, A + 8 * S, 0)),
        check=lambda a: len(tags(a, "L")) == 2)
    # --- ordered: ties in arrival order, a queue across activations, never a merge
    add("ordered_ties_running", spec_("running", ordered=True, sides=2, gap=S, wait=5 * S),
        Steps().batch((1, A + 3 * S, 0), (1, A + S, 1), (1, A + S, 0), (1, A + 3 * S, 1), (1, A + S, 0), (1, A + 9 * S, 0))
        .batch((1, A + 30 * S, 1)))
    add("ordered_queue_complete", spec_("complete", ordered=True, sides=2, gap=2 * S, wait=4 * S),
        Steps().batch((1, A + 6 * S, 0), (1, A + 2 * S, 1)).batch((1, A + 7 * S, 1), (1, A + 3 * S, 0))
        .batch((1, A + 9 * S, 0)).batch((1, A + 15 * S, 1), (2, A, 0)))
    add("ordered_final_four_sides", spec_("final", ordered=True, sides=4, gap=S, wait=S),
        Steps().batch((1, A, 3), (1, A + S, 1), (2, A, 0), (2, A + 1, 2), (2, A + 2, 3), (2, A + 3, 1), (1, A + 2, 1))
        .batch((1, A + 50 * S, 0)))
    # --- notify under a stepping clock, then EOF
    sc = Steps(now=A)
    for i, k in enumerate((1, 2, 1, 1, 2, 1)):
        t = A + i * 3 * S
        sc.batch((k, t, i % 2), (k, t + 1, (i + 1) % 2), (k, t + 2, 0), now=t)
        if i % 2:
            sc.notify(t + 2 * S)
    add("stepping_clock_notify_running", spec_("running", ordered=True, sides=2, gap=2 * S, wait=0), sc.notify(A + 60 * S))
    add("stepping_clock_notify_final", spec_("final", ordered=False, sides=2, gap=2 * S, wait=S), sc)
    add("eof_closes_open_sessions", spec_("final", ordered=False, sides=3, gap=S, wait=F),
        Steps().batch((1, A + 9 * S, 2), (1, A + 1 * S, 0), (1, A + 5 * S, 1)).batch((1, A, 1), (2, A + 3 * S, 0), (1, A + 2 * S, 2)),
        check=lambda a: not any(a[:-1]) and len(tags(a, "M")) == 4)

    seeded = {}
    for seed in sp.SEEDED:
        spec, steps = sp.seeded_steps(seed, moving=seed % 3 != 0)
        acts, stats = run_reference(spec, steps)
        assert not (spec["ordered"] and stats["merges"]), seed  # ordered mode never merges
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts], merges=stats["merges"],
                                      chains=stats["chains"])
    path = os.path.join(ROOT, "tests", "golden", "session_product_join_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
