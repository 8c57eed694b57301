"""Generate ``tests/golden/join_window_cases.json`` from the UNMODIFIED reference `join_window`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_join_window_golden.py

Every case builds a real reference flow (``win.join_window`` over an ``EventClock`` and a ``TumblingWindower`` or
``SlidingWindower``), pulls the ``stateful_batch`` step's builder out of the step tree, and drives the reference's own
``_WindowLogic`` + ``_SlidingWindowerLogic`` + ``_JoinWindowLogic`` with the engine rules of src/operators.rs:755-806
(ascending key string per activation; a logic that reports itself empty is discarded, clock state included), :808-858
(notify: every key whose ``notify_at()`` has come) and :862-894 (EOF).

Items are ``(key_str, (value, ts_us))`` on side ``side``; values are distinct ints, so they double as the handles the
device joins.  Hand-built cases store their rows in full; the seeded streams of ``tests/join_window_oracle.py``
(``seeded_steps``) store the SHA-256 of their rows.  The file holds data only.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import join_window_oracle as jo  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A = jo.S, jo.A
UTC_MAX = 253_402_300_799_999_999


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def join_builder(spec, now_getter):
    """The reference's `stateful_batch` builder of a `join_window` flow; side values are ``(value, ts_us)``."""
    wait = timedelta.max if spec["wait_us"] == jo.WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda v: dt(v[1]), wait_for_system_duration=wait, now_getter=now_getter)
    align = dt(spec["align_us"])
    length, offset = (timedelta(microseconds=spec["length_us"]), timedelta(microseconds=spec["offset_us"]))
    if spec["length_us"] == spec["offset_us"]:
        windower = win.TumblingWindower(length=length, align_to=align)
    else:
        windower = win.SlidingWindower(length=length, offset=offset, align_to=align)
    flow = Dataflow("g")
    sides = [op.input(f"in{i}", flow, TestingSource([])) for i in range(spec["sides"])]
    win.join_window("j", clock, windower, *sides, insert_mode=spec["insert_mode"], emit_mode=spec["emit_mode"],
                    ordered=spec["ordered"])
    return refstub.find_stateful_batch(flow).builder


def run_reference(spec, steps):
    now = [dt(steps[0][1])]
    builder = join_builder(spec, lambda: now[0])
    logics, acts = {}, []

    def conv(ks, events):
        rows = []
        for wid, tag, p in events:
            if tag == "E":
                rows.append([int(ks), wid, "E", [None if v is None else v[0] for v in p]])
            elif tag == "L":
                rows.append([int(ks), wid, "L", [p[0], p[1][0]]])
            else:
                rows.append([int(ks), wid, "M", [us(p.open_time), us(p.close_time)]])
        return rows

    def done_with(ks, res, rows):
        events, done = res
        rows.extend(conv(ks, list(events)))
        if done:
            del logics[ks]  # src/operators.rs:796-799

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
    return acts


def spec_(ins="last", emit="final", ordered=True, sides=2, length=10 * S, offset=None, align=A, wait=0):
    return dict(insert_mode=ins, emit_mode=emit, ordered=ordered, sides=sides, length_us=length,
                offset_us=length if offset is None else offset, align_us=align, wait_us=wait)


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

    def add(name, spec, st, check=None, cite=None):
        acts = run_reference(spec, st.steps)
        if check is not None:
            assert check(acts), (name, acts)
        cases[name] = dict(spec=spec, steps=st.steps, acts=acts, cite=cite)

    def tags(acts, tag):
        return [r for act in acts for r in act if r[2] == tag]

    # docs/guide/concepts/joins.md:470-634: two users, 1 h tumbling windows from 2023-01-01, wait 0; the reference
    # emits (456: 8328, (Hive, None)), (123: 8328, (Bee, bee@)), (456: 8329, (None, hive@))
    g0 = us(datetime(2023, 12, 14, tzinfo=timezone.utc))
    H = 3600 * S
    add("guide_walkthrough_tumbling", spec_(length=H, align=us(datetime(2023, 1, 1, tzinfo=timezone.utc))),
        Steps().batch((123, g0, 0), (456, g0, 0)).batch((123, g0 + H // 4, 1), (456, g0 + 5 * H // 4, 1)),
        check=lambda a: [[r[0], r[1]] for r in tags(a, "E")] == [[456, 8328], [123, 8328], [456, 8329]],
        cite="docs/guide/concepts/joins.md:470-634")
    # --- insert and emit modes -----------------------------------------------------------------------------------------
    add("first_complete_refills", spec_("first", "complete", wait=jo.WAIT_FOREVER),
        Steps().batch((1, A, 0), (1, A + 1, 0), (1, A + 2, 1), (1, A + 3, 1), (1, A + 4, 0), (1, A + 5, 1), (1, A + 6, 1)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2], [4, 3]])
    add("last_final_overwrites", spec_("last", "final", wait=jo.WAIT_FOREVER),
        Steps().batch((1, A, 0), (1, A + 1, 0), (1, A + 2, 1)).batch((1, A + 3, 1), (1, A + 4, 0), (2, A, 1)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[4, 3], [None, 5]])
    add("running_every_value", spec_("first", "running", wait=2 * S),
        Steps().batch((1, A, 1), (1, A + 1, 1), (1, A + 2, 0), (1, A + 3, 0)).batch((1, A + 20 * S, 1)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[None, 0], [None, 0], [2, 0], [2, 0], [None, 4]])
    # --- window geometry -----------------------------------------------------------------------------------------------
    add("sliding_indivisible_offset", spec_("last", "final", sides=2, length=7 * S, offset=3 * S, align=A + 1, wait=S),
        Steps().batch((1, A, 0), (1, A + 4 * S, 1), (1, A + 9 * S, 0)).batch((1, A + 30 * S, 1)))
    add("negative_window_ids", spec_("first", "final", sides=2, length=4 * S, offset=2 * S, align=A + 100 * S, wait=0),
        Steps().batch((3, A + 93 * S, 0), (3, A + 95 * S, 1), (3, A + 99 * S, 0)).batch((3, A + 100 * S + 1, 1)),
        check=lambda a: any(r[1] < 0 for r in tags(a, "M")))
    add("late_sliding_all_windows", spec_("last", "running", sides=2, length=6 * S, offset=2 * S, wait=0),
        Steps().batch((5, A + 20 * S, 0)).batch((5, A + 11 * S, 1), (5, A + 19 * S, 0), (5, A + 21 * S, 1)),
        check=lambda a: len(tags(a, "L")) == 6)
    # unordered: the higher window opens first, so it closes (and is reported) first
    add("close_first_opened_not_id_order", spec_("last", "final", ordered=False, sides=2, length=5 * S, wait=20 * S),
        Steps().batch((1, A + 12 * S, 0), (1, A + 2 * S, 1), (1, A + 7 * S, 0)).batch((1, A + 40 * S, 1)),
        check=lambda a: [r[1] for r in tags(a, "M")][:3] == [2, 0, 1])
    # --- ordered mode ----------------------------------------------------------------------------------------------------
    add("ordered_ties_stable", spec_("last", "running", ordered=True, sides=2, wait=5 * S),
        Steps().batch((1, A + 3 * S, 0), (1, A + S, 1), (1, A + S, 0), (1, A + 3 * S, 1), (1, A + S, 0), (1, A + 9 * S, 0))
        .batch((1, A + 30 * S, 1)))
    add("ordered_queue_across_activations", spec_("first", "complete", ordered=True, sides=2, wait=4 * S),
        Steps().batch((1, A + 6 * S, 0), (1, A + 2 * S, 1)).batch((1, A + 7 * S, 1), (1, A + 3 * S, 0))
        .batch((1, A + 9 * S, 0)).batch((1, A + 15 * S, 1), (2, A, 0)))
    # queue[0] (ts A+8) is not the smallest queued ts (A+5): the notify wakes at A+8 once `now` drifts the watermark
    add("ordered_notify_wakes_queue_head", spec_("last", "final", ordered=True, sides=2, length=20 * S, wait=10 * S),
        Steps(now=A).batch((4, A + 8 * S, 0), (4, A + 5 * S, 1), (4, A + 12 * S, 1), now=A)
        .notify(A + 4 * S).notify(A + 8 * S).notify(A + 9 * S).notify(A + 30 * S))
    add("wait_forever_flush_at_eof", spec_("last", "final", ordered=True, sides=3, length=4 * S, wait=jo.WAIT_FOREVER),
        Steps().batch((1, A + 9 * S, 2), (1, A + 1 * S, 0), (1, A + 5 * S, 1)).batch((1, A, 1), (2, A + 3 * S, 0), (1, A + 2 * S, 2)),
        check=lambda a: not any(a[:-1]) and len(tags(a, "M")) == 4)
    # --- discard: an empty logic goes, clock included; the next item starts from UTC_MIN again -----------------------
    add("discard_resets_watermark", spec_("last", "final", ordered=False, sides=2, length=5 * S, wait=0),
        Steps(now=A).batch((1, A + 20 * S, 0), now=A).notify(A + 10 * S).batch((1, A + 2 * S, 1), now=A + 10 * S)
        .batch((1, A + 1 * S, 0)).notify(A + 30 * S).batch((1, A, 0), now=A + 30 * S),
        check=lambda a: len(tags(a, "L")) == 1 and len(tags(a, "M")) == 3)
    # --- side counts ------------------------------------------------------------------------------------------------------
    add("one_side", spec_("first", "complete", ordered=False, sides=1, length=3 * S, wait=S),
        Steps().batch((1, A, 0), (1, A + 1, 0), (2, A + S, 0)).batch((1, A + 10 * S, 0)))
    add("four_sides_partial", spec_("last", "final", ordered=True, sides=4, length=10 * S, wait=S),
        Steps().batch((1, A, 3), (1, A + S, 1), (2, A, 0), (2, A + 1, 2), (2, A + 2, 3), (2, A + 3, 1)).batch((1, A + 50 * S, 0)))
    # --- clocks -----------------------------------------------------------------------------------------------------------
    # SystemClock: every item is stamped with the batch's system time and the wait is 0
    sc = Steps(now=A)
    for i, k in enumerate((1, 2, 1, 1, 2, 1)):
        now = A + i * 3 * S
        sc.batch((k, now, i % 2), (k, now, (i + 1) % 2), now=now)
        if i % 2:
            sc.notify(now + 2 * S)
    add("system_clock_moving_now", spec_("last", "running", ordered=True, sides=2, length=5 * S, wait=0), sc.notify(A + 60 * S))
    add("near_utc_max", spec_("last", "final", ordered=True, sides=2, length=10 * S, align=0, wait=0),
        Steps().batch((1, UTC_MAX - 25 * S, 0), (2, UTC_MAX - 12 * S, 1)).batch((1, UTC_MAX - 19 * S - 1, 1), (2, UTC_MAX - 11 * S, 0)))
    add("moving_clock_drift_late", spec_("first", "complete", ordered=False, sides=2, length=4 * S, wait=2 * S),
        Steps(now=A + S).batch((7, A + S, 0), (8, A + S, 1), now=A + S).batch((7, A + 2 * S, 1), now=A + 21 * S)
        .batch((8, A + 25 * S, 0), now=A + 22 * S).notify(A + 40 * S))
    # --- keys whose decimal text orders differently from their value -------------------------------------------------------
    keys = [0, 2**64 - 1, 2**63] + [10**k - 1 for k in range(1, 20)] + [10**k for k in range(1, 20)]
    add("digit_boundary_keys", spec_("last", "running", ordered=False, sides=2, length=S, wait=0),
        Steps().batch(*[(k, A + (i % 3) * S, i % 2) for i, k in enumerate(keys)]).batch(*[(k, A + 5 * S, 1) for k in keys[::-1]]))

    seeded = {}
    for seed in jo.SEEDED:
        spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
        acts = run_reference(spec, steps)
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts])
    path = os.path.join(ROOT, "tests", "golden", "join_window_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
