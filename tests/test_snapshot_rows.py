"""`bytewax_b200.snapshot_rows`: the columnar device snapshot turned into the reference's per-key `_WindowSnapshot` objects.

The reference's OWN classes produced tests/golden/snapshot_cases.json (oracle/gen_golden.py main_snapshots): a stream folded
by the real `_WindowLogic` objects up to a cut, what each key's `snapshot()` holds there, and what the uninterrupted logics
emit after it.  Here the state at the cut is written the way the device dumps it (one row per live (key, pane): what
`bw_snapshot_take` returns), converted, compared with the reference's snapshots field by field, handed to this package's
window logic as `resume_state`, and the resumed logics must emit exactly what the reference's uninterrupted ones did."""
import json
import math
import os
import pickle
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

from oracle import streams

ALIGN = 1_640_995_200_000_000
S = 1_000_000
I64_MIN = -(1 << 63)
EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
NOW = datetime(2030, 1, 1, tzinfo=timezone.utc)  # the frozen system clock of oracle/gen_golden.py


def _us(d):
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def _dt(us):
    return EPOCH + timedelta(microseconds=us)


def _count_builder(spec):
    """The `stateful_batch` builder of this package's `count_window` for `spec` (items are (key_str, value, ts_us))."""
    from bytewax_b200 import operators as op
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.operators import windowing as win
    from bytewax_b200.testing import TestingSource

    clock = win.EventClock(lambda x: _dt(x[2]), wait_for_system_duration=timedelta(microseconds=spec["wait_us"]), now_getter=lambda: NOW)
    windower = win.SlidingWindower(length=timedelta(microseconds=spec["length_us"]),
                                   offset=timedelta(microseconds=spec["offset_us"] or spec["length_us"]), align_to=_dt(spec["align_us"]))
    flow = Dataflow("g")
    win.count_window("w", op.input("in", flow, TestingSource([])), clock, windower, lambda x: x[0])
    stack = list(flow.substeps)
    while stack:
        step = stack.pop(0)
        if type(step).__name__ == "stateful_batch":
            return step.builder
        stack = list(getattr(step, "substeps", [])) + stack
    raise LookupError("no stateful_batch step")


def _device_columns(accepted, opened_by_key, max_ts, red, length, offset, closed_upto):
    """What the table holds at the cut: per key the live panes (those under a still-open window) with the fold of the
    accepted items in them, the first arrival index per pane, the key's running maximum and its `closed_upto`."""
    g = math.gcd(length, offset)
    a, b = offset // g, length // g
    cols = {n: [] for n in ("key", "pane_id", "acc", "count", "open_seq", "max_ts_us", "closed_upto")}
    fold = {"count": lambda x, v: x + 1, "sum": lambda x, v: x + v, "min": min, "max": max}[red]
    for k, opened in opened_by_key.items():
        panes = {}
        for seq, ts, v in accepted[k]:
            q = (ts - ALIGN) // g
            w_lo, w_hi = -((-(q - b + 1)) // a), q // a
            if not any(w in opened for w in range(w_lo, w_hi + 1)):
                continue  # every window of this pane has closed: the pane is gone
            cur = panes.get(q)
            if cur is None:
                panes[q] = [(1 if red == "count" else v), seq]
            else:
                cur[0] = fold(cur[0], v)
        for q, (acc, seq) in sorted(panes.items()):
            cols["key"].append(k)
            cols["pane_id"].append(q)
            cols["acc"].append(acc & 0xFFFFFFFFFFFFFFFF)
            cols["count"].append(0)
            cols["open_seq"].append(seq)
            cols["max_ts_us"].append(max_ts[k])
            cols["closed_upto"].append(closed_upto.get(k, I64_MIN))
    dt = dict(key=np.uint64, pane_id=np.int64, acc=np.uint64, count=np.uint64, open_seq=np.uint64, max_ts_us=np.int64, closed_upto=np.int64)
    return {n: np.array(v, dtype=dt[n]) for n, v in cols.items()}


@pytest.mark.parametrize("red,length,offset,wait", streams.SNAPSHOT_CASES)
def test_resume_on_the_reference_logic(red, length, offset, wait, golden_dir):
    from bytewax_b200 import snapshot_rows
    from bytewax_b200.operators import windowing as win

    with open(os.path.join(golden_dir, "snapshot_cases.json")) as f:
        case = json.load(f)[f"{red}-{length}-{offset}-{wait}"]
    spec, batches, cut = streams.snapshot_case(red, length, offset, wait)
    off = spec["offset_us"] or spec["length_us"]
    ref = case["keys"]
    # the reference's state at the cut: accepted items (all but the dropped ones), newest timestamps, open windows (in
    # first-opened order)
    accepted = {int(ks): [(sq, t, v) for sq, (t, v) in streams.key_items(batches[:cut], int(ks)).items() if sq not in c["dropped"]]
                for ks, c in ref.items()}
    max_ts = {k: max(t for _sq, t, _v in items) for k, items in accepted.items()}
    opened_by_key = {int(ks): {w: None for w, *_ in c["opened"]} for ks, c in ref.items()}
    closed_upto = {}
    for k, opened in opened_by_key.items():
        # sliding windows: every id below the oldest open one that covers a live pane has been emitted
        closed_upto[k] = min(opened) - 1 if (offset and opened) else I64_MIN
    cols = _device_columns(accepted, opened_by_key, max_ts, red, spec["length_us"], off, closed_upto)
    assert len(cols["key"]) > 5
    snaps = snapshot_rows.window_snapshots(cols, reduction=red, length_us=spec["length_us"], offset_us=off, align_us=ALIGN,
                                           wait_us=wait * S, now_us=_us(NOW), frozen_now_us=_us(NOW), classes=win)
    assert set(snaps) == set(ref)
    for ks, real in ref.items():
        mine = snaps[ks]
        # same windows with the same bounds, in the same (first-opened) order
        assert [[w, _us(m.open_time), _us(m.close_time), sorted(m.merged_ids)] for w, m in mine.windower_state.opened.items()] == real["opened"], ks
        assert dict((w, v) for w, v in real["logic_states"]) == mine.logic_states, ks
        assert _us(mine.clock_state.watermark_base) - _us(mine.clock_state.system_time_of_max_event) == real["clock_diff_us"], ks
    rows = snapshot_rows.recovery_rows("flow.step", snaps, 7)
    assert all(isinstance(pickle.loads(r[3]), win._WindowSnapshot) for r in rows) and [r[1] for r in rows] == sorted(snaps)
    if red == "count":  # (for reduce / max the reference's accumulator is the ITEM; a number resumes count and numeric folds only)
        builder, unwrap = _count_builder(spec), (lambda acc: acc)
        resumed = {ks: builder(pickle.loads(pickle.dumps(s))) for ks, s in snaps.items()}
        got = streams.drive(resumed, builder, batches[cut:], unwrap, cut)
        got_eof = [(ks, w, tag, unwrap(p) if tag == "E" else None) for ks in sorted(resumed) for w, tag, p in resumed[ks].on_eof()[0] if tag != "M"]
        assert [list(r) for r in got] == case["want"] and [list(r) for r in got_eof] == case["want_eof"]
