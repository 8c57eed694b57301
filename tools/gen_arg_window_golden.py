"""Generate ``tests/golden/arg_window_cases.json`` from the UNMODIFIED reference `max_window` / `min_window` with `by=`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_arg_window_golden.py

Every case builds a real reference flow (``win.max_window`` / ``win.min_window`` with ``by=lambda e: e[2]`` over an
``EventClock`` and a tumbling, sliding or session windower), pulls the ``stateful_batch`` step's builder out of the
step tree, and drives the reference's own ``_WindowLogic`` + windower + ``_FoldWindowLogic`` with the engine rules of
src/operators.rs:755-806 (ascending key string per activation, discard of logics that report themselves empty),
:808-858 (notify: every key whose ``notify_at()`` has come) and :862-894 (EOF).

Items are ``(handle, ts_us, by)``; rows name items by handle.  By-values are ints or floats; floats are stored as
``float.hex`` strings so NaN and -0.0 survive JSON.  Hand-built cases store their rows in full; the seeded streams of
``tests/arg_window_oracle.py`` (``seeded_steps``) store the SHA-256 of their rows.  The file holds data only.
"""

import json
import math
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import arg_window_oracle as aw  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A = aw.S, aw.A
UTC_MAX = 253_402_300_799_999_999
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def arg_builder(spec, now_getter):
    """The reference's `stateful_batch` builder of a `max_window` / `min_window` flow over items ``(handle, ts, by)``."""
    wait = timedelta.max if spec["wait_us"] == aw.WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda e: dt(e[1]), wait_for_system_duration=wait, now_getter=now_getter)
    if "gap_us" in spec:
        windower = win.SessionWindower(gap=timedelta(microseconds=spec["gap_us"]))
    else:
        align = dt(spec["align_us"])
        length, offset = timedelta(microseconds=spec["length_us"]), timedelta(microseconds=spec["offset_us"])
        if spec["length_us"] == spec["offset_us"]:
            windower = win.TumblingWindower(length=length, align_to=align)
        else:
            windower = win.SlidingWindower(length=length, offset=offset, align_to=align)
    flow = Dataflow("g")
    up = op.input("in", flow, TestingSource([]))
    getattr(win, f"{spec['extreme']}_window")("a", up, clock, windower, by=lambda e: e[2])
    return refstub.find_stateful_batch(flow).builder


def run_reference(spec, steps):
    now = [dt(steps[0][1])]
    builder = arg_builder(spec, lambda: now[0])
    logics, acts = {}, []

    def conv(ks, events):
        rows = []
        for wid, tag, p in events:
            if tag in ("E", "L"):
                rows.append([int(ks), wid, tag, p[0]])
            elif "gap_us" in spec:
                rows.append([int(ks), wid, "M", [us(p.open_time), us(p.close_time), sorted(p.merged_ids)]])
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
            for k, t, b, h in zip(step[2], step[3], step[4], step[5]):
                grouped.setdefault(str(k), []).append((h, t, aw.dec(b)))
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


def tw(ext="max", length=10 * S, offset=None, align=A, wait=0):
    return dict(extreme=ext, length_us=length, offset_us=length if offset is None else offset, align_us=align, wait_us=wait)


def sw(ext="max", gap=10 * S, wait=0):
    return dict(extreme=ext, gap_us=gap, wait_us=wait)


class Steps:
    """Builds golden steps; every item gets a fresh handle."""

    def __init__(self, now=A + 10**6 * S):
        self.steps, self.n, self.now = [], 0, now

    def batch(self, *items, now=None):
        """``items``: ``(key, ts, by)``."""
        if now is not None:
            self.now = now
        k, t, b = ([it[i] for it in items] for i in range(3))
        self.steps.append(["batch", self.now, k, t, [aw.enc(x) for x in b], list(range(self.n, self.n + len(items)))])
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

    def picks(acts):
        return [r[3] for act in acts for r in act if r[2] == "E"]

    def tags(acts, tag):
        return [r for act in acts for r in act if r[2] == tag]

    F = aw.WAIT_FOREVER
    nan, inf = math.nan, math.inf
    # --- the reference's own tests: pytests/operators/windowing/test_max_min_window.py (tumbling 10 s, wait 0)
    T0 = us(datetime(2022, 1, 1, tzinfo=timezone.utc))
    ref = "pytests/operators/windowing/test_max_min_window.py"
    ref_items = [(0, T0, 1), (0, T0 + 4 * S, 9), (0, T0 + 8 * S, 3), (0, T0 + 12 * S, 10), (0, T0 + 13 * S, 4)]
    add("ref_max_window", tw("max", align=T0), Steps().batch(*ref_items), check=lambda a: picks(a) == [1, 3], cite=ref + ":14-44")
    add("ref_min_window", tw("min", align=T0), Steps().batch(*ref_items), check=lambda a: picks(a) == [0, 4], cite=ref + ":47-77")
    # --- ties: the earlier item stays, in every window and for both extremes
    for ext in ("max", "min"):
        add(f"ties_keep_first_{ext}", tw(ext, wait=F), Steps().batch((1, A, 5), (1, A + S, 5), (1, A + 2 * S, 7), (1, A + 3 * S, 7),
                                                                      (1, A + 4 * S, 5)).batch((1, A + 5 * S, 7), (1, A + 6 * S, 5)),
            check=lambda a, e=ext: picks(a) == ([2] if e == "max" else [0]))
        add(f"sliding_ties_{ext}", tw(ext, length=6 * S, offset=2 * S, wait=F),
            Steps().batch(*[(2, A + i * S, (i % 3) * 1.5) for i in range(12)]))
    # --- +-0.0 ties: -0.0 first keeps its place against +0.0 and the other way round
    add("signed_zero_ties_max", tw("max", wait=F), Steps().batch((3, A, -0.0), (3, A + S, 0.0), (4, A, 0.0), (4, A + S, -0.0)),
        check=lambda a: picks(a) == [0, 2])
    add("signed_zero_ties_min", tw("min", wait=F), Steps().batch((3, A, 0.0), (3, A + S, -0.0), (4, A, -0.0), (4, A + S, 0.0)),
        check=lambda a: picks(a) == [0, 2])
    # --- NaN: a NaN pick is never beaten; a NaN value never wins
    for ext in ("max", "min"):
        add(f"nan_first_{ext}", tw(ext, wait=F), Steps().batch((5, A, nan), (5, A + S, 5.0), (5, A + 2 * S, -inf), (5, A + 3 * S, inf)),
            check=lambda a: picks(a) == [0])
        add(f"nan_later_{ext}", tw(ext, wait=F), Steps().batch((6, A, 1.0), (6, A + S, nan), (6, A + 2 * S, 2.0), (6, A + 3 * S, nan)))
    # --- +-inf and subnormals
    add("inf_subnormal_max", tw("max", wait=F),
        Steps().batch((7, A, -inf), (7, A + S, -5e-324), (7, A + 2 * S, 5e-324), (7, A + 3 * S, 0.0), (8, A, inf), (8, A + S, inf)),
        check=lambda a: picks(a) == [2, 4])
    add("inf_subnormal_min", tw("min", wait=F),
        Steps().batch((7, A, inf), (7, A + S, 5e-324), (7, A + 2 * S, -5e-324), (7, A + 3 * S, -0.0), (8, A, -inf), (8, A + S, -inf)),
        check=lambda a: picks(a) == [2, 4])
    # --- i64 extremes (and neighbours that would tie in f64)
    for ext in ("max", "min"):
        add(f"i64_extremes_{ext}", tw(ext, wait=F),
            Steps().batch((9, A, 0), (9, A + S, I64_MIN), (9, A + 2 * S, I64_MAX), (9, A + 3 * S, I64_MIN), (9, A + 4 * S, I64_MAX),
                          (10, A, (1 << 53) + 1), (10, A + S, 1 << 53), (10, A + 2 * S, (1 << 53) + 2), (10, A + 3 * S, -(1 << 53) - 1)))
    # --- sliding: one value is the pick in some of its windows only (6 s / 2 s: each value in 3 windows)
    add("sliding_pick_in_some_windows", tw("max", length=6 * S, offset=2 * S, wait=F),
        Steps().batch((11, A, 9), (11, A + 3 * S, 5), (11, A + 5 * S, 7), (11, A + 7 * S, 6)).batch((11, A + 9 * S, 8)))
    add("sliding_replaced_everywhere", tw("min", length=6 * S, offset=2 * S, align=A + 1, wait=S),
        Steps().batch((12, A + 2 * S, 5), (12, A + 3 * S, 4), (12, A + 4 * S, 3)).batch((12, A + 20 * S, 0)))
    # --- late items with wait > 0: one late row per window of late_for(ts)
    add("late_with_wait", tw("max", length=6 * S, offset=2 * S, wait=2 * S),
        Steps().batch((13, A + 10 * S, 1), (13, A + 3 * S, 4), (13, A + 8 * S, 2), (13, A + 20 * S, 3), (13, A + 17 * S, 9)),
        check=lambda a: len(tags(a, "L")) >= 3)
    add("session_late_with_wait", sw("min", gap=S, wait=2 * S),
        Steps().batch((13, A + 10 * S, 1), (13, A + 3 * S, 4), (13, A + 8 * S, 2), (13, A + 20 * S, 3), (13, A + 17 * S, 9)),
        check=lambda a: [r[1] for r in tags(a, "L")] == [-1, -1])
    # --- a moving clock: the watermark drifts with `now`, and notify closes windows without new items
    add("moving_clock_notify", tw("max", wait=S),
        Steps(now=A).batch((14, A + S, 3), (15, A + 2 * S, 1), now=A).notify(A + 5 * S).batch((14, A + 3 * S, 9), now=A + 8 * S)
        .notify(A + 12 * S).batch((15, A + 25 * S, 2), now=A + 14 * S).notify(A + 40 * S))
    add("session_moving_clock_notify", sw("max", gap=2 * S, wait=S),
        Steps(now=A).batch((14, A + S, 3), (15, A + 2 * S, 1), now=A).notify(A + 3 * S).notify(A + 6 * S)
        .batch((14, A + 3 * S, 9), now=A + 8 * S).notify(A + 40 * S))
    # --- discard and reopen: a notify closes key 16's last window and the logic goes with its clock; A+5 s, late for
    # the old clock, then opens a new window 0
    add("discard_and_reopen", tw("max", length=10 * S, wait=0),
        Steps(now=A).batch((16, A + S, 4), (16, A + 12 * S, 1), now=A).notify(A + 20 * S).batch((16, A + 5 * S, 8), (16, A + 6 * S, 8)),
        check=lambda a: not tags(a, "L") and [r[1] for r in tags(a, "E")] == [0, 1, 0])
    # --- sessions: session 0 (A+10, h0 by 5) merges into session 1 (opened at A), whose pick h2 (by 5) arrived AFTER
    # h0; the tie keeps the survivor's pick, so the rule is not "earliest arrival wins"
    add("merge_survivor_wins_tie_with_later_pick", sw("max", gap=2 * S, wait=F),
        Steps().batch((17, A + 10 * S, 5), (17, A, 1), (17, A + S, 5), (17, A + 5 * S, 0), (17, A + 8 * S, 0), (17, A + 3 * S, 0),
                      (17, A + 6 * S, 0)),
        check=lambda a: picks(a) == [2] and [r[1] for r in tags(a, "M")] == [1])
    # the merged-away session's pick is strictly better: it replaces the survivor's
    add("merge_orig_strictly_better", sw("min", gap=3 * S, wait=F),
        Steps().batch((18, A, 5), (18, A + 6 * S, 1), (18, A + 3 * S, 7)), check=lambda a: picks(a) == [1])
    # --- a value played into a session that a merge just took away: A+10 extends session 0 (A+20) to A+10, which then
    # merges into session 1 (A); the value still goes to session 0, whose pick then meets session 1's in the merge
    add("value_into_merged_away_session", sw("max", gap=10 * S, wait=F),
        Steps().batch((19, A + 20 * S, 4), (19, A, 2), (19, A + 10 * S, 9)), check=lambda a: picks(a) == [2])
    add("value_into_merged_away_session_loses", sw("max", gap=10 * S, wait=F),
        Steps().batch((19, A + 20 * S, 4), (19, A, 2), (19, A + 10 * S, 3)), check=lambda a: picks(a) == [0])
    # --- a chain of merges in one call: three sessions, then two bridges into session 0 (a NaN in between)
    add("merge_chain_one_call", sw("max", gap=2 * S, wait=F),
        Steps().batch((20, A, 1.0), (20, A + 4 * S, 3.0), (20, A + 8 * S, 2.0), (20, A + 2 * S, nan), (20, A + 6 * S, 3.0)),
        check=lambda a: picks(a) == [4] and len(tags(a, "M")) == 1)
    # session 0 absorbs session 1, then is itself merged into session 2 in the same call (merged ids: direct only)
    add("merge_chain_survivor_merged_away", sw("max", gap=4 * S, wait=F),
        Steps().batch((26, A + 10 * S, 5), (26, A + 15 * S, 9), (26, A + 3 * S, 1), (26, A + 12 * S, 2), (26, A + 7 * S, 3)),
        check=lambda a: picks(a) == [1] and [r[3][2] for r in tags(a, "M")] == [[0]])
    add("merge_chain_across_calls", sw("min", gap=2 * S, wait=F),
        Steps().batch((21, A, 4), (21, A + 4 * S, 2), (21, A + 8 * S, 3)).batch((21, A + 2 * S, 9), (21, A + 6 * S, 1)))
    # --- sessions kept open at EOF near UTC_MAX: close >= UTC_MAX - gap stays open
    add("session_eof_near_utc_max", sw("max", gap=2 * S, wait=0),
        Steps().batch((22, UTC_MAX - S, 1), (23, UTC_MAX - 3 * S, 2), (24, UTC_MAX - 2 * S, 3)),
        check=lambda a: [r[0] for r in tags(a, "M")] == [23])
    # --- SystemClock-like: every item at the batch's system time, wait 0
    sc = Steps(now=A)
    for i, k in enumerate((25, 26, 25, 25, 26, 25)):
        now = A + i * 3 * S
        sc.batch((k, now, i % 3), (k, now, 2 - i % 3), now=now)
        if i % 2:
            sc.notify(now + 2 * S)
    add("system_clock_moving_now", tw("min", length=4 * S, wait=0), sc.notify(A + 60 * S))
    # --- keys whose decimal text orders differently from their value
    keys = [0, 2**64 - 1, 2**63] + [10**k - 1 for k in range(1, 20)] + [10**k for k in range(1, 20)]
    add("digit_boundary_keys", tw("max", length=5 * S, offset=S, wait=0),
        Steps().batch(*[(k, A + (i % 3) * S, i % 4) for i, k in enumerate(keys)]).batch(*[(k, A + 9 * S, 1) for k in keys[::-1]]))

    seeded = {}
    for seed in aw.SEEDED:
        spec, steps = aw.seeded_steps(seed, moving=seed % 3 != 1)
        acts = run_reference(spec, steps)
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts])
    path = os.path.join(ROOT, "tests", "golden", "arg_window_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
