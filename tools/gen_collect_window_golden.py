"""Generate ``tests/golden/collect_window_cases.json`` from the UNMODIFIED reference `collect_window`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_collect_window_golden.py

Every case builds a real reference flow (``win.collect_window`` into ``list`` over an ``EventClock`` and a
``TumblingWindower`` or ``SlidingWindower``), pulls the ``stateful_batch`` step's builder out of the step tree, and
drives the reference's own ``_WindowLogic`` + ``_SlidingWindowerLogic`` + ``_FoldWindowLogic`` with the collect
callbacks, under the engine rules of src/operators.rs:755-806 (ascending key string per activation; a logic that
reports itself empty is discarded, clock state included), :808-858 (notify: every key whose ``notify_at()`` has come)
and :862-894 (EOF).

Items are ``(key_str, (value, ts_us))``; values are distinct ints, so they double as the handles the device collects.
Steps use ``tests/join_window_oracle.py``'s format with one side.  Hand-built cases store their rows in full; the
seeded streams of ``tests/collect_window_oracle.py`` (``seeded_steps``) store the SHA-256 of their rows.  The file holds
data only.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import collect_window_oracle as co  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A = co.S, co.A
UTC_MAX = 253_402_300_799_999_999


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def collect_builder(spec, now_getter):
    """The reference's `stateful_batch` builder of a `collect_window` flow; values are ``(value, ts_us)``."""
    wait = timedelta.max if spec["wait_us"] == co.WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda v: dt(v[1]), wait_for_system_duration=wait, now_getter=now_getter)
    align = dt(spec["align_us"])
    length, offset = (timedelta(microseconds=spec["length_us"]), timedelta(microseconds=spec["offset_us"]))
    if spec["length_us"] == spec["offset_us"]:
        windower = win.TumblingWindower(length=length, align_to=align)
    else:
        windower = win.SlidingWindower(length=length, offset=offset, align_to=align)
    flow = Dataflow("g")
    up = op.input("in", flow, TestingSource([]))
    win.collect_window("c", up, clock, windower, into=list, ordered=spec["ordered"])
    return refstub.find_stateful_batch(flow).builder


def run_reference(spec, steps):
    now = [dt(steps[0][1])]
    builder = collect_builder(spec, lambda: now[0])
    logics, acts = {}, []

    def conv(ks, events):
        rows = []
        for wid, tag, p in events:
            if tag == "E":
                rows.append([int(ks), wid, "E", [v[0] for v in p]])
            elif tag == "L":
                rows.append([int(ks), wid, "L", p[0]])
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
            for k, t, v in zip(step[2], step[3], step[5]):
                grouped.setdefault(str(k), []).append((v, t))
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


def spec_(ordered=True, length=10 * S, offset=None, align=A, wait=0):
    return dict(ordered=ordered, length_us=length, offset_us=length if offset is None else offset, align_us=align, wait_us=wait)


class Steps:
    """Builds golden steps; every value is a fresh int (its handle)."""

    def __init__(self, now=A + 10**6 * S):
        self.steps, self.n, self.now = [], 0, now

    def batch(self, *items, now=None):
        """``items``: ``(key, ts)``."""
        if now is not None:
            self.now = now
        k, t = ([it[i] for it in items] for i in range(2))
        self.steps.append(["batch", self.now, k, t, [0] * len(items), list(range(self.n, self.n + len(items)))])
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

    # pytests/operators/windowing/test_collect_window.py: one key, 10 s tumbling windows from 2022-01-01, wait forever,
    # ordered, one item per activation at +0, +8, +4, +13, +12: played in ts order at EOF, [0, 2, 1] then [4, 3]
    add("reference_test_stream", spec_(wait=co.WAIT_FOREVER),
        Steps().batch((1, A)).batch((1, A + 8 * S)).batch((1, A + 4 * S)).batch((1, A + 13 * S)).batch((1, A + 12 * S)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2, 1], [4, 3]],
        cite="pytests/operators/windowing/test_collect_window.py")
    # the operator's docstring (windowing.py:1436-1576): 10 s tumbling from 2023-01-01, two keys, wait 0
    d0 = us(datetime(2023, 1, 1, tzinfo=timezone.utc))
    add("docstring_example", spec_(length=10 * S, align=d0),
        Steps().batch((1, d0 + 1 * S), (2, d0 + 2 * S), (1, d0 + 5 * S), (1, d0 + 11 * S), (2, d0 + 15 * S)),
        check=lambda a: len(tags(a, "M")) == 4)
    # --- window geometry -----------------------------------------------------------------------------------------------
    add("sliding_indivisible_offset", spec_(length=7 * S, offset=3 * S, align=A + 1, wait=S),
        Steps().batch((1, A), (1, A + 4 * S), (1, A + 9 * S)).batch((1, A + 30 * S)))
    add("negative_window_ids", spec_(length=4 * S, offset=2 * S, align=A + 100 * S, wait=0),
        Steps().batch((3, A + 93 * S), (3, A + 95 * S), (3, A + 99 * S)).batch((3, A + 100 * S + 1)),
        check=lambda a: any(r[1] < 0 for r in tags(a, "M")))
    add("late_sliding_all_windows", spec_(length=6 * S, offset=2 * S, wait=0),
        Steps().batch((5, A + 20 * S)).batch((5, A + 11 * S), (5, A + 19 * S), (5, A + 21 * S)),
        check=lambda a: len(tags(a, "L")) == 6)
    # unordered: the higher window opens first, so it closes (and is reported) first
    add("close_first_opened_not_id_order", spec_(ordered=False, length=5 * S, wait=20 * S),
        Steps().batch((1, A + 12 * S), (1, A + 2 * S), (1, A + 7 * S)).batch((1, A + 40 * S)),
        check=lambda a: [r[1] for r in tags(a, "M")][:3] == [2, 0, 1])
    # --- ordered mode ----------------------------------------------------------------------------------------------------
    add("ordered_ties_stable", spec_(ordered=True, wait=5 * S),
        Steps().batch((1, A + 3 * S), (1, A + S), (1, A + S), (1, A + 3 * S), (1, A + S), (1, A + 9 * S)).batch((1, A + 30 * S)),
        check=lambda a: tags(a, "E")[0][3] == [1, 2, 4, 0, 3, 5])
    add("ordered_queue_across_activations", spec_(ordered=True, wait=4 * S),
        Steps().batch((1, A + 6 * S), (1, A + 2 * S)).batch((1, A + 7 * S), (1, A + 3 * S))
        .batch((1, A + 9 * S)).batch((1, A + 15 * S), (2, A)))
    # queue[0] (ts A+8) is not the smallest queued ts (A+5): the notify wakes at A+8 once `now` drifts the watermark
    add("ordered_notify_wakes_queue_head", spec_(ordered=True, length=20 * S, wait=10 * S),
        Steps(now=A).batch((4, A + 8 * S), (4, A + 5 * S), (4, A + 12 * S), now=A)
        .notify(A + 4 * S).notify(A + 8 * S).notify(A + 9 * S).notify(A + 30 * S))
    add("wait_forever_flush_at_eof", spec_(ordered=True, length=4 * S, wait=co.WAIT_FOREVER),
        Steps().batch((1, A + 9 * S), (1, A + 1 * S), (1, A + 5 * S)).batch((1, A), (2, A + 3 * S), (1, A + 2 * S)),
        check=lambda a: not any(a[:-1]) and len(tags(a, "M")) == 4)
    # --- discard: an empty logic goes, clock included; the next item starts from UTC_MIN again -----------------------
    add("discard_resets_watermark", spec_(ordered=False, length=5 * S, wait=0),
        Steps(now=A).batch((1, A + 20 * S), now=A).notify(A + 10 * S).batch((1, A + 2 * S), now=A + 10 * S)
        .batch((1, A + 1 * S)).notify(A + 30 * S).batch((1, A), now=A + 30 * S),
        check=lambda a: len(tags(a, "L")) == 1 and len(tags(a, "M")) == 3)
    # --- clocks -----------------------------------------------------------------------------------------------------------
    # SystemClock: every item is stamped with the batch's system time and the wait is 0
    sc = Steps(now=A)
    for i, k in enumerate((1, 2, 1, 1, 2, 1)):
        now = A + i * 3 * S
        sc.batch((k, now), (k, now), now=now)
        if i % 2:
            sc.notify(now + 2 * S)
    add("system_clock_moving_now", spec_(ordered=True, length=5 * S, wait=0), sc.notify(A + 60 * S))
    add("near_utc_max", spec_(ordered=True, length=10 * S, align=0, wait=0),
        Steps().batch((1, UTC_MAX - 25 * S), (2, UTC_MAX - 12 * S)).batch((1, UTC_MAX - 19 * S - 1), (2, UTC_MAX - 11 * S)))
    add("moving_clock_drift_late", spec_(ordered=False, length=4 * S, wait=2 * S),
        Steps(now=A + S).batch((7, A + S), (8, A + S), now=A + S).batch((7, A + 2 * S), now=A + 21 * S)
        .batch((8, A + 25 * S), now=A + 22 * S).notify(A + 40 * S))
    # --- keys whose decimal text orders differently from their value -------------------------------------------------------
    keys = [0, 2**64 - 1, 2**63] + [10**k - 1 for k in range(1, 20)] + [10**k for k in range(1, 20)]
    add("digit_boundary_keys", spec_(ordered=False, length=S, wait=0),
        Steps().batch(*[(k, A + (i % 3) * S) for i, k in enumerate(keys)]).batch(*[(k, A + 5 * S) for k in keys[::-1]]))

    seeded = {}
    for seed in co.SEEDED:
        spec, steps = co.seeded_steps(seed, moving=seed % 3 != 0)
        acts = run_reference(spec, steps)
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts])
    path = os.path.join(ROOT, "tests", "golden", "collect_window_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
