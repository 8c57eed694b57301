"""Generate ``tests/golden/session_cases.json`` from the UNMODIFIED reference session windower.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_session_golden.py

Every case builds a real reference flow (``win.count_window`` / ``win.reduce_window`` / ``win.max_window`` /
``win.min_window`` over an ``EventClock`` and a ``SessionWindower``), pulls the ``stateful_batch`` step's builder out of
the step tree, and drives the reference's own ``_WindowLogic`` + ``_SessionWindowerLogic`` with the engine rules of
src/operators.rs:755-806 (ascending key string per activation), :808-858 (notify: every key whose ``notify_at()`` has
come) and :862-894 (EOF).  Session state is never discarded (windowing.py:798-806).

Hand-built cases store their rows in full; the seeded streams of ``tests/session_oracle.py`` (``seeded_steps``) store
the SHA-256 of their rows, as tests/golden/live_reference_cases.json does for the sliding windower.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import session_oracle as so  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A = so.S, so.A
UTC_MAX = 253_402_300_799_999_999


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def session_builder(spec, now_getter):
    """The reference's `stateful_batch` builder for a session fold; items are ``(key_str, value, ts_us)``."""
    wait = timedelta.max if spec["wait_us"] == so.WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda x: dt(x[2]), wait_for_system_duration=wait, now_getter=now_getter)
    windower = win.SessionWindower(gap=timedelta(microseconds=spec["gap_us"]))
    flow = Dataflow("g")
    s = op.input("in", flow, TestingSource([]))
    red = spec["reduction"]
    if red == "count":
        win.count_window("w", s, clock, windower, lambda x: x[0])
        unwrap = lambda acc: acc  # noqa: E731
    else:
        keyed = op.key_on("k", s, lambda x: x[0])
        if red == "sum":  # operator.add on the values: fold `acc + v`, merge `into + orig`
            win.reduce_window("w", keyed, clock, windower, lambda a, b: (a[0], a[1] + b[1], b[2]))
        elif red == "max":
            win.max_window("w", keyed, clock, windower, by=lambda x: x[1])
        elif red == "min":
            win.min_window("w", keyed, clock, windower, by=lambda x: x[1])
        else:
            raise ValueError(red)
        unwrap = lambda acc: acc[1]  # noqa: E731
    return refstub.find_stateful_batch(flow).builder, unwrap


def run_reference_sessions(spec, steps):
    now = [dt(steps[0][1])]
    builder, unwrap = session_builder(spec, lambda: now[0])
    logics, acts = {}, []

    def conv(ks, events):
        rows = []
        for wid, tag, p in events:
            if tag == "E":
                rows.append([int(ks), wid, "E", unwrap(p)])
            elif tag == "L":
                rows.append([int(ks), wid, "L", p[1]])
            else:
                rows.append([int(ks), wid, "M", [us(p.open_time), us(p.close_time), sorted(p.merged_ids)]])
        return rows

    for step in steps:
        now[0] = dt(step[1])
        rows = []
        if step[0] == "batch":
            grouped = {}
            for k, t, v in zip(step[2], step[3], step[4]):
                grouped.setdefault(str(k), []).append((str(k), v, t))
            for ks in sorted(grouped):
                logic = logics.get(ks)
                if logic is None:
                    logic = logics[ks] = builder(None)
                events, done = logic.on_batch(grouped[ks])
                rows.extend(conv(ks, list(events)))
                assert not done  # windowing.py:798-806
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now[0]:
                    events, _ = logics[ks].on_notify()
                    rows.extend(conv(ks, list(events)))
        acts.append(rows)
    rows = []
    for ks in sorted(logics):
        events, _ = logics[ks].on_eof()
        rows.extend(conv(ks, list(events)))
    acts.append(rows)
    return acts


def spec_(red="count", gap=5 * S, wait=0, dtype="i64"):
    return dict(reduction=red, val_dtype=dtype, gap_us=gap, wait_us=wait)


def frozen(*batches, now=A + 10**9 * S):
    """Activations on a frozen system clock: ``(keys, ts, vals)`` each."""
    return [["batch", now, list(k), list(t), list(v)] for k, t, v in batches]


def one_key(ts, vals=None, key=0, per_activation=1):
    vals = vals if vals is not None else [1] * len(ts)
    return [([key] * len(ts[i : i + per_activation]), ts[i : i + per_activation], vals[i : i + per_activation])
            for i in range(0, len(ts), per_activation)]


def main():
    cases = {}

    def add(name, spec, steps, expect_down=None, cite=None, min_merges=0):
        acts = run_reference_sessions(spec, steps)
        merges = sum(len(r[3][2]) for act in acts for r in act if r[2] == "M")
        assert merges >= min_merges, (name, merges, min_merges)  # a case named for merges must really merge
        if expect_down is not None:
            down = [[r[0], r[1], r[3]] for act in acts for r in act if r[2] == "E"]
            assert down == expect_down, (name, down, expect_down)
        cases[name] = dict(spec=spec, steps=steps, acts=acts, cite=cite)

    # --- the reference's own tests --------------------------------------------------------------------------------
    add("ref_fold_window_session", spec_("count", 5 * S),
        frozen(*one_key([A + s * S for s in (1, 5, 11, 12, 13, 14, 20, 1)])),
        expect_down=[[0, 0, 2], [0, 1, 4], [0, 2, 1]], cite="pytests/operators/windowing/test_fold_window.py:97-140")
    # pytests/operators/windowing/test_session_windower.py:19-127 (open_for shapes; gap 10 s, wait keeps all on time)
    for name, secs in (("ref_extend_forward", (0, 5)), ("ref_extend_forward_exact_gap", (0, 10)),
                       ("ref_extend_backward", (0, -5)), ("ref_extend_backward_exact_gap", (0, -10)),
                       ("ref_extend_merge", (0, 20, 10)), ("ref_within_existing", (0, 10, 5))):
        add(name, spec_("count", 10 * S, so.WAIT_FOREVER), frozen(*one_key([A + s * S for s in secs])),
            cite="pytests/operators/windowing/test_session_windower.py:19-127")
    # :160-265 _session_find_merges shapes, reached through open_for: multi (1,0),(2,0); no-yes-no (2,1)
    add("ref_find_merges_multi", spec_("count", 10 * S, so.WAIT_FOREVER),
        frozen(*one_key([A + 0 * S, A + 30 * S, A + 15 * S, A + 5 * S, A + 10 * S], per_activation=5)),
        cite="pytests/operators/windowing/test_session_windower.py:210-237")
    add("ref_find_merges_no_yes_no", spec_("count", 10 * S, so.WAIT_FOREVER),
        frozen(*one_key([A + 0 * S, A + 20 * S, A + 40 * S, A + 32 * S, A + 25 * S], per_activation=5)),
        cite="pytests/operators/windowing/test_session_windower.py:240-265")
    # :268-293 SystemClock: every item is stamped with the batch's system time (wait 0)
    add("ref_session_with_system_clock", spec_("count", 10 * S),
        [["batch", A, [0] * 10, [A] * 10, list(range(10))]], expect_down=[[0, 0, 10]],
        cite="pytests/operators/windowing/test_session_windower.py:268-293")

    # --- gap edges ------------------------------------------------------------------------------------------------
    add("gap_exact_both_sides", spec_("sum", 2 * S, so.WAIT_FOREVER),
        frozen(*one_key([A, A + 2 * S, A - 2 * S, A + 4 * S + 1, A - 4 * S - 1], [1, 2, 3, 4, 5], per_activation=5)))
    add("gap_zero", spec_("count", 0), frozen(*one_key([A, A, A + 1, A + 1, A + 3, A + 2, A + 2], per_activation=7),
                                               ([1, 1], [A + 10, A + 11], [0, 0])))
    add("gap_zero_wait", spec_("max", 0, 5), frozen(*one_key([A + 10, A + 8, A + 4, A + 10, A + 20, A + 14], [1, 5, 3, 9, 2, 7],
                                                         per_activation=2)))
    # --- first session by id wins; merge into the earlier-opened one --------------------------------------------------
    # sessions 0 [A+20], 1 [A+0]; A+10 is within gap of both: session 0 (first id) takes it, opens at A+10 and then
    # merges into session 1 (opened earlier) -- the survivor is 1, the item's value sits in 0 until the merge pass
    add("first_by_id_merge_into_earlier", spec_("sum", 10 * S, so.WAIT_FOREVER),
        frozen(*one_key([A + 20 * S, A, A + 10 * S, A + 35 * S], [100, 10, 1, 1000], per_activation=4)))
    # A+13 is 7 s before session 0 (id 0) and 5 s after session 1: the first by id takes it, not the nearest, and its
    # value reaches session 1 through the merge: 0.1 + (0.2 + 0.3) = 0.6, where the nearest would give 0.6000000000000001
    add("first_by_id_not_nearest", spec_("sum", 7 * S, so.WAIT_FOREVER, "f64"),
        frozen(*one_key([A + 20 * S, A + 8 * S, A + 13 * S], [0.2, 0.1, 0.3], per_activation=3)), min_merges=1,
        expect_down=[[0, 1, 0.6]])
    # --- 3-way and chained merges; a survivor merged later; merged sessions closing in the same activation -----------
    # sessions 12 s apart, gap 6 s: an item 6 s after a session's close extends it to within the gap of the next one
    # (`_session_find_merges` merges at exactly `gap`).  One activation, two merges into session 0: {1, 2}
    add("three_way_merge", spec_("count", 6 * S, so.WAIT_FOREVER),
        frozen(*one_key([A, A + 12 * S, A + 24 * S, A + 6 * S, A + 18 * S], per_activation=5)), min_merges=2)
    # 2 absorbs 3, then 1 absorbs 2 (1 holds {2}, not 3), then 0 absorbs 1 -- all in one activation; next, a NEW session
    # 4 opened 5 s before 0 absorbs 0 (the survivor is the earliest opened, not the lowest id, and the item that
    # extended 0 is folded into 0 before the merge pass); session 4 closes two activations later holding {0}
    add("chained_merges_survivor_merged_later", spec_("sum", 6 * S, 100 * S),
        frozen(*one_key([A + 30 * S, A + 42 * S, A + 54 * S, A + 66 * S], [1, 2, 4, 8], per_activation=4),
               ([0] * 3, [A + 60 * S, A + 48 * S, A + 36 * S], [16, 32, 64]),
               ([0] * 2, [A + 20 * S, A + 25 * S], [128, 256]),
               ([0], [A + 200 * S], [512])), min_merges=1, expect_down=[[0, 4, 511], [0, 5, 512]])
    # the second activation merges 3 into 2 and then closes 0 (merged {1}) and 2 (merged {3}) in the same pass
    add("merged_close_same_activation", spec_("count", 4 * S, 10 * S),
        frozen(([0, 0, 0], [A, A + 8 * S, A + 4 * S], [0, 0, 0]), ([0, 0, 0, 0], [A + 40 * S, A + 48 * S, A + 44 * S, A + 70 * S], [0, 0, 0, 0])),
        min_merges=2)
    # --- lates: wait 0, wait > 0, wait forever --------------------------------------------------------------------
    for w, tag in ((0, "wait0"), (3 * S, "wait3"), (so.WAIT_FOREVER, "wait_forever")):
        add(f"lates_{tag}", spec_("min", 2 * S, w),
            frozen(([0, 1, 0, 1], [A + 10 * S, A + 10 * S, A + 5 * S, A + 8 * S], [5, 6, 7, 8]),
                   ([0, 0, 1, 1, 0], [A + 9 * S, A + 30 * S, A + 6 * S, A + 7 * S, A + 29 * S], [-1, -2, -3, -4, -5]),
                   ([1, 0], [A + 31 * S, A + 26 * S], [9, 9])))
    # --- time range edges -----------------------------------------------------------------------------------------
    add("before_1970", spec_("sum", 2 * S, S),
        frozen(*one_key([-5 * S, -4 * S, -1, 0, -9 * S, 3 * S, -20 * S], [1, 2, 3, 4, 5, 6, 7], per_activation=3)))
    add("near_utc_max", spec_("count", 10 * S, 0),
        frozen(([0, 1, 2], [UTC_MAX - 30 * S, UTC_MAX - 10 * S, UTC_MAX - 10 * S - 1], [0, 0, 0]),
               ([3], [UTC_MAX - 10 * S + 1], [0])))
    # --- keys whose decimal text orders differently from their value ---------------------------------------------------
    keys = [0, 2**64 - 1, 2**63] + [10**k - 1 for k in range(1, 20)] + [10**k for k in range(1, 20)]
    add("digit_boundary_keys", spec_("count", 1 * S, 0),
        frozen((keys, [A + (i % 3) * S for i in range(len(keys))], [0] * len(keys)),
               (keys[::-1], [A + 5 * S] * len(keys), [0] * len(keys)),
               (keys[:5], [A + 20 * S] * 5, [0] * 5)))
    # --- f64: sums whose bits depend on the merge order; signed zeros and NaN in max / min -----------------------------
    add("f64_sum_merge_order", spec_("sum", 6 * S, so.WAIT_FOREVER, "f64"),
        frozen(*one_key([A, A + 12 * S, A + 24 * S, A + 1 * S, A + 13 * S, A + 25 * S, A + 6 * S, A + 18 * S],
                        [1e16, 1.0, -1e16, 1.0, 0.1, 1.0, 0.2, 0.3], per_activation=8),
               *one_key([A + 100 * S, A + 112 * S, A + 106 * S], [0.3, 0.1, 0.2], per_activation=3)), min_merges=3)
    # (merging as found would give 2.3 and 0.6000000000000001 where the reference's order gives 2.0 and 0.6)
    for red in ("max", "min"):
        add(f"f64_{red}_signed_zero_nan", spec_(red, 6 * S, so.WAIT_FOREVER, "f64"),
            frozen(*one_key([A, A + 1, A + 2, A + 3], [0.0, -0.0, 0.0, -0.0], key=1, per_activation=4),
                   *one_key([A, A + 1, A + 2], [-0.0, 0.0, -0.0], key=2, per_activation=3),
                   *one_key([A, A + 1, A + 2], [float("nan"), 1.0, -1.0], key=3, per_activation=3),
                   *one_key([A, A + 1, A + 2], [1.0, float("nan"), 2.0], key=4, per_activation=3),
                   # merges: into (opened first) vs orig, with zeros and NaN on either side
                   ([5, 5, 5], [A, A + 12 * S, A + 6 * S], [0.0, -0.0, -0.0]),
                   ([6, 6, 6], [A, A + 12 * S, A + 6 * S], [-0.0, 0.0, 0.0]),
                   ([7, 7, 7], [A, A + 12 * S, A + 6 * S], [float("nan"), 3.0, 3.0]),
                   ([8, 8, 8], [A, A + 12 * S, A + 6 * S], [3.0, float("nan"), float("nan")]),
                   ([9, 9, 9, 9], [A, A, A + 12 * S, A + 6 * S], [2.0, 2.0, 2.0, 2.0])), min_merges=5)
    # --- moving clock with notify steps ---------------------------------------------------------------------------
    add("moving_clock_notify", spec_("count", 2 * S, S),
        [["batch", A + 1 * S, [1, 1, 2], [A, A + 1 * S, A + 1 * S], [0, 0, 0]],
         ["notify", A + 2 * S], ["notify", A + 4 * S], ["notify", A + 5 * S],
         ["batch", A + 6 * S, [1, 3], [A + 5 * S, A + 5 * S], [0, 0]],
         ["notify", A + 9 * S], ["notify", A + 30 * S]])
    add("moving_clock_drift_late", spec_("sum", 3 * S, 2 * S),
        [["batch", A + 1 * S, [7, 8], [A + 1 * S, A + 1 * S], [5, 6]],
         ["batch", A + 21 * S, [7], [A + 2 * S], [100]],
         ["batch", A + 22 * S, [8], [A + 25 * S], [7]],
         ["notify", A + 40 * S]])

    seeded = {}
    for seed in so.SEEDED:
        spec, steps = so.seeded_steps(seed, moving=seed % 3 != 0)
        acts = run_reference_sessions(spec, steps)
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts])
    path = os.path.join(ROOT, "tests", "golden", "session_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
