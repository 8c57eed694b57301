"""The same flows as tests/test_api_engine.py with the CUDA path enabled (run_main(..., gpu=True)):
the recogniser hands numeric windowed folds to libbwgpu; rows must equal the host engine's.  -m gpu."""

import operator
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.inputs import KeyedColumns  # noqa: E402
from bytewax_b200.operators.windowing import ZERO_TD, EventClock, SlidingWindower, TumblingWindower  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)


def _both(build):
    outs = []
    for gpu in (False, True):
        flow, sinks = build()
        run_main(flow, gpu=gpu)
        outs.append(sinks)
    return outs


def test_count_window_reference_expectation_on_gpu():
    # pytests/operators/windowing/test_count_window.py:10-35
    inp = [{"time": ALIGN + timedelta(seconds=s), "user": u, "val": 1} for s, u in ((0, "a"), (4, "a"), (8, "b"), (12, "a"), (13, "a"))]

    def build():
        out, meta = [], []
        flow = Dataflow("test_df")
        s = op.input("inp", flow, TestingSource(inp))
        wo = win.count_window("add", s, EventClock(lambda e: e["time"], ZERO_TD, now_getter=lambda: FROZEN),
                              TumblingWindower(timedelta(seconds=10), ALIGN), lambda e: e["user"])
        op.output("out", wo.down, TestingSink(out))
        op.output("meta", wo.meta, TestingSink(meta))
        return flow, (out, meta)

    host, gpu = _both(build)
    assert gpu[0] == [("a", (0, 2)), ("a", (1, 2)), ("b", (0, 1))]
    assert gpu == host


def test_sliding_sum_with_late_items_matches_host():
    rnd = np.random.default_rng(3)
    n = 3000
    ts = ALIGN + np.array([timedelta(seconds=float(i * 0.05 + rnd.uniform(-4, 4))) for i in range(n)])
    items = [(f"k{int(rnd.integers(0, 20))}", (t, int(rnd.integers(-50, 50)))) for t in ts]

    class N(int):
        pass

    def num(v):
        x = N(v[1])
        x.ts = v[0]
        return x

    def build():
        out, late = [], []
        flow = Dataflow("df")
        s = op.input("inp", flow, TestingSource(items, batch_size=97))
        nums = op.map_value("num", s, num)
        wo = win.reduce_window("sum", nums, EventClock(lambda v: v.ts, timedelta(seconds=1), now_getter=lambda: FROZEN),
                               SlidingWindower(timedelta(seconds=10), timedelta(seconds=5), ALIGN), operator.add)
        op.output("out", wo.down, TestingSink(out))
        op.output("late", wo.late, TestingSink(late))
        return flow, (out, late)

    host, gpu = _both(build)
    assert [(k, (w, int(v))) for k, (w, v) in gpu[0]] == [(k, (w, int(v))) for k, (w, v) in host[0]]
    assert [(k, (w, int(v))) for k, (w, v) in gpu[1]] == [(k, (w, int(v))) for k, (w, v) in host[1]]
    assert len(gpu[1]) > 0 and len(gpu[0]) > 50


def test_columnar_source_feeds_the_cuda_fold():
    """A source yielding KeyedColumns: one epoch == one activation, no per-item Python objects."""
    A_US = 1_640_995_200_000_000
    n = 200_000
    batches = []
    for b in range(5):
        i = np.arange(b * n, (b + 1) * n)
        batches.append(("cols", KeyedColumns(keys=(i * 2654435761 % 1000).astype(np.uint64), ts_us=(A_US + i * 100).astype(np.int64))))
    out = []
    flow = Dataflow("df")
    s = op.input("inp", flow, TestingSource(batches))
    # A frozen system clock: with wait 0, the watermark would otherwise advance with the wall time between activations, and
    # a key's next event (100 ms of event time later) would be late whenever the host took longer than that between them.
    clock = EventClock(lambda v: None, ZERO_TD, now_getter=lambda: FROZEN)
    # already keyed columns: count_window's key_on would call key() per item, so use fold_window's plan via count on keyed input
    wo = win.fold_window("sum", s, clock, TumblingWindower(timedelta(seconds=10), ALIGN), lambda: 0,
                         lambda a, _: a + 1, lambda a, b: a + b, ordered=False,
                         _gpu_plan=win.GpuFoldPlan("count", clock, TumblingWindower(timedelta(seconds=10), ALIGN), False, lambda v: v))
    op.output("out", wo.down, TestingSink(out))
    run_main(flow, gpu=True)
    total = sum(c for _k, (_w, c) in out)
    assert total == 5 * n
    wids = sorted({w for _k, (w, _c) in out})
    assert wids == list(range(10))  # 1e6 events x 100 us = 100 s -> windows 0..9
    first_epoch_keys = [k for k, (w, _c) in out if w == 0]
    assert first_epoch_keys == sorted(first_epoch_keys)  # ascending key-string order within an activation


def test_final_folds_on_gpu_match_the_reference_expectations():
    # pytests/operators/test_count_final.py:6-16, test_reduce_final.py:6-17, test_max_min_final.py (sorted-key EOF order)
    def build():
        outs = [[], [], [], []]
        flow = Dataflow("test_df")
        s = op.input("inp", flow, TestingSource(["a", "a", "b", "c", "b", "a"]))
        op.output("o0", op.count_final("count", s, lambda x: x), TestingSink(outs[0]))
        nums = op.input("nums", flow, TestingSource([("b", 7), ("a", 1), ("a", 8), ("10", 1), ("9", 2), ("b", -3), ("a", 5)]))
        op.output("o1", op.reduce_final("sum", nums, operator.add), TestingSink(outs[1]))
        op.output("o2", op.max_final("max", nums), TestingSink(outs[2]))
        op.output("o3", op.min_final("min", nums), TestingSink(outs[3]))
        return flow, outs

    host, gpu = _both(build)
    assert gpu[0] == [("a", 3), ("b", 2), ("c", 1)]
    assert gpu[1] == [("10", 1), ("9", 2), ("a", 14), ("b", 4)]
    assert gpu[2] == [("10", 1), ("9", 2), ("a", 8), ("b", 7)]
    assert gpu[3] == [("10", 1), ("9", 2), ("a", 1), ("b", -3)]
    assert gpu == host


def test_final_fold_large_against_numpy():
    """count/sum/max per key over 3 activations of 2^20 rows through the C ABI (ts_source == BW_TS_NONE)."""
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    rnd = np.random.default_rng(3)
    n, nk = 1 << 20, 50_000
    for red in ("count", "sum", "max", "min"):
        fold = gpu.WindowFold(ctx, red, val_dtype="i64", final=True, capacity_hint=nk, max_batch_rows=n, max_emit_rows=nk + 16)
        allk, allv = [], []
        for _ in range(3):
            k = rnd.integers(0, nk, n).astype(np.uint64)
            v = rnd.integers(-1000, 1000, n)
            fold.ingest(k, None if red == "count" else v)
            assert fold.advance().closed_key.size == 0  # nothing is emitted before EOF
            allk.append(k)
            allv.append(v)
        em = fold.eof()
        k, v = np.concatenate(allk), np.concatenate(allv)
        order = np.argsort(k, kind="stable")
        uk, start = np.unique(k[order], return_index=True)
        if red == "count":
            want = np.diff(np.append(start, k.size))
        else:
            want = {"sum": np.add, "max": np.maximum, "min": np.minimum}[red].reduceat(v[order], start)
        got = dict(zip(em.closed_key.tolist(), em.closed_acc.astype(np.int64).tolist()))
        assert got == dict(zip(uk.tolist(), want.tolist())), red
        assert em.closed_key.tolist() == sorted(uk.tolist(), key=str)  # ascending key-string order
        assert set(em.closed_window_id.tolist()) == {0}
        fold.close()
    ctx.close()


def test_max_min_window_numeric_on_gpu():
    # the shape of pytests/operators/windowing/test_max_min_window.py:14-67 with numeric values (the recogniser's domain):
    # values 1, 9, 3 in window 0 and 10, 4 in window 1
    class N(int):
        pass

    def num(val, sec):
        x = N(val)
        x.ts = ALIGN + timedelta(seconds=sec)
        return x

    inp = [("a", num(1, 0)), ("a", num(9, 4)), ("a", num(3, 8)), ("a", num(10, 12)), ("a", num(4, 13))]

    def build():
        outs = [[], []]
        flow = Dataflow("test_df")
        s = op.input("inp", flow, TestingSource(inp))
        clock = EventClock(lambda v: v.ts, ZERO_TD, now_getter=lambda: FROZEN)
        windower = TumblingWindower(timedelta(seconds=10), ALIGN)
        op.output("o0", win.max_window("max", s, clock, windower).down, TestingSink(outs[0]))
        op.output("o1", win.min_window("min", s, clock, windower).down, TestingSink(outs[1]))
        return flow, outs

    host, gpu = _both(build)
    assert [(k, (w, int(v))) for k, (w, v) in gpu[0]] == [("a", (0, 9)), ("a", (1, 10))]
    assert [(k, (w, int(v))) for k, (w, v) in gpu[1]] == [("a", (0, 1)), ("a", (1, 4))]
    assert [[(k, (w, int(v))) for k, (w, v) in o] for o in host] == [[(k, (w, int(v))) for k, (w, v) in o] for o in gpu]


def test_stateful_map_detector_runs_on_k5():
    """`op.stateful_map` with the declared z-score detector (BASELINE config C2's mapper, examples/anomaly_detector.py) is
    handed to bw_smap_* by the recogniser; items must equal the host engine's, which calls the mapper per item."""
    from bytewax_b200 import engine
    from bytewax_b200.detectors import ZScoreDetector

    rnd = np.random.default_rng(5)
    n = 20_000
    vals = rnd.normal(10.0, 2.0, n)
    vals[rnd.random(n) < 0.01] += 25.0  # anomalies
    items = [(f"m{int(k)}", float(v)) for k, v in zip(rnd.integers(0, 300, n), vals)]
    made = []
    orig = engine._gpu_step_for

    def spy(step_id, plan):
        st = orig(step_id, plan)
        made.append(type(st).__name__)
        return st

    def build():
        out = []
        flow = Dataflow("test_df")
        s = op.input("inp", flow, TestingSource(items, batch_size=2500))
        d = op.stateful_map("detector", s, ZScoreDetector(window=10, threshold_z=2.0))
        op.output("out", d, TestingSink(out))
        return flow, out

    engine._gpu_step_for = spy
    try:
        host, gpu = _both(build)
    finally:
        engine._gpu_step_for = orig
    assert made == ["_GpuSmapStep"]
    assert len(gpu) == n and any(r[1][3] for r in gpu)
    # key order, values, means and flags are identical (K5 sums in CPython's order: compensated, newest first); sigma is
    # a correctly rounded sqrt on the device and `x ** 0.5` (libm pow, not always correctly rounded) in the mapper: 1 ulp
    assert [(k, v[0], v[1], v[3]) for k, v in gpu] == [(k, v[0], v[1], v[3]) for k, v in host]
    assert np.allclose([v[2] for _k, v in gpu], [v[2] for _k, v in host], rtol=1e-15, atol=0.0)


@pytest.mark.parametrize("insert_mode,emit_mode", [("last", "complete"), ("first", "final"), ("last", "running")])
def test_join_runs_on_k6(insert_mode, emit_mode):
    """Two-sided `op.join` on bw_join_* (values travel as handles): rows and their order equal the host `_JoinLogic`."""
    from bytewax_b200 import engine

    rnd = np.random.default_rng(9)
    n = 6000
    left = [(f"u{int(k)}", {"name": f"n{i}"}) for i, k in enumerate(rnd.integers(0, 1500, n))]
    right = [(f"u{int(k)}", ("mail", i)) for i, k in enumerate(rnd.integers(0, 1500, n))]
    made = []
    orig = engine._gpu_step_for

    def spy(step_id, plan):
        st = orig(step_id, plan)
        made.append(type(st).__name__)
        return st

    def build():
        out = []
        flow = Dataflow("test_df")
        a = op.input("a", flow, TestingSource(left, batch_size=500))
        b = op.input("b", flow, TestingSource(right, batch_size=500))
        j = op.join("j", a, b, insert_mode=insert_mode, emit_mode=emit_mode)
        op.output("out", j, TestingSink(out))
        return flow, out

    engine._gpu_step_for = spy
    try:
        host, gpu = _both(build)
    finally:
        engine._gpu_step_for = orig
    assert made == ["_GpuJoinStep"]
    assert len(gpu) > 0
    assert gpu == host


def _moving_clock_flow(gpu):
    S = timedelta(seconds=1)
    now_box = [ALIGN]
    # (key, event time, system time of arrival, value)
    raw = [("a", 1.0, 2.0, 5), ("a", 1.5, 2.0, 6), ("b", 1.8, 2.5, 1), ("c", 9.5, 9.6, 1), ("c", 11.0, 10.0, 2),
           ("z", 12.0, 13.0, 100), ("z", 14.0, 15.0, 200),
           ("a", 3.0, 16.0, 7),   # a's logic was discarded when its window closed: accepted again (a fresh watermark)
           ("c", 12.0, 16.5, 4),  # c's window 1 is still open; maximum 11 seen at system time 10 -> watermark 17.5: LATE by drift alone
           ("z", 27.0, 27.5, 300), ("b", 26.0, 28.0, 2)]
    items = [(k, (ALIGN + ev * S, ALIGN + sy * S, v)) for k, ev, sy, v in raw]

    def tick(kv):
        now_box[0] = kv[1][1]  # the system clock reads the item's arrival time from here on
        return kv

    out, late = [], []
    flow = Dataflow("test_df")
    s = op.input("inp", flow, TestingSource(items, batch_size=1))
    s = op.map("tick", s, tick)
    clock = EventClock(lambda e: e[0], ZERO_TD, now_getter=lambda: now_box[0])
    windower = TumblingWindower(timedelta(seconds=10), ALIGN)
    wo = win.fold_window("sum", s, clock, windower, lambda: 0, lambda a, e: a + e[2], operator.add, ordered=False,
                         _gpu_plan=win.GpuFoldPlan("sum", clock, windower, False, lambda e: e[2]))
    op.output("out", wo.down, TestingSink(out))
    # (the CUDA path's late stream carries the numeric projection of the value, the host's the item itself)
    op.output("late", op.map_value("lv", wo.late, lambda wv: (wv[0], wv[1][2] if isinstance(wv[1], tuple) else wv[1])), TestingSink(late))
    run_main(flow, gpu=gpu)
    return out, late


def test_idle_key_closes_when_the_system_clock_moves():
    """EventClock with a moving `now_getter`: the watermark drifts with the system clock (windowing.py:263-302) and the
    notify phase closes an idle key's window before EOF (src/operators.rs:808-858) -- on the CUDA path as on the host."""
    host = _moving_clock_flow(False)
    # window 0 of a, b and c closes while only z is receiving items; c's last item is late although it is its key's newest
    assert host[0][:3] == [("c", (0, 1)), ("a", (0, 11)), ("b", (0, 1))], host[0]
    assert host[1] == [("c", (1, 4))], host[1]
    assert _moving_clock_flow(True) == host


def test_system_clock_windows_on_gpu(monkeypatch):
    """SystemClock (windowing.py:190-222): timestamp == watermark == system time.  On the CUDA path it is an event clock
    whose timestamps are the arrival times with wait 0, windows closing as the system clock passes them (notify phase)."""
    S = timedelta(seconds=1)
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0, 1), ("b", 2.0, 1), ("a", 3.0, 1), ("z", 12.0, 1), ("a", 14.0, 1), ("z", 31.0, 1), ("b", 33.0, 1)]
    items = [(k, (ALIGN + sy * S, v)) for k, sy, v in raw]

    def tick(kv):
        now_box[0] = kv[1][0]
        return kv

    outs = []
    for gpu in (False, True):
        now_box[0] = ALIGN
        out = []
        flow = Dataflow("test_df")
        s = op.input("inp", flow, TestingSource(items, batch_size=1))
        s = op.map("tick", s, tick)
        wo = win.count_window("cnt", s, win.SystemClock(), TumblingWindower(timedelta(seconds=10), ALIGN), lambda kv: kv[0])
        op.output("out", wo.down, TestingSink(out))
        run_main(flow, gpu=gpu)
        outs.append(out)
    assert outs[0][:2] == [("a", (0, 2)), ("b", (0, 1))]  # closed when the clock read 12 s, long before EOF
    assert outs[1] == outs[0]


@pytest.mark.parametrize("red", ["count", "sum", "min"])
def test_fold_columns_public_operator(red):
    """`win.fold_columns`: KeyedColumns batches in, one activation each on the CUDA path, rows equal the host engine's
    (which expands the columns into items); with `columns_out=True` the output streams carry WindowColumns."""
    A_US = 1_640_995_200_000_000
    n = 100_000
    rnd = np.random.default_rng(17)
    batches = []
    for b in range(4):
        i = np.arange(b * n, (b + 1) * n)
        ts = A_US + i * 100 + rnd.integers(-3_000_000, 3_000_000, n)  # disorder beyond the 1 s wait: some rows are late
        batches.append(KeyedColumns(keys=(i * 2654435761 % 3000).astype(np.uint64), ts_us=ts.astype(np.int64),
                                    vals=None if red == "count" else rnd.integers(-50, 50, n).astype(np.int64)))

    def build(columns_out):
        out, late, meta = [], [], []
        flow = Dataflow("df")
        s = op.input("inp", flow, TestingSource(batches))
        wo = win.fold_columns("fold", s, red, SlidingWindower(timedelta(seconds=10), timedelta(seconds=5), ALIGN), timedelta(seconds=1),
                              columns_out=columns_out, now_getter=lambda: FROZEN)
        op.output("out", wo.down, TestingSink(out))
        op.output("late", wo.late, TestingSink(late))
        op.output("meta", wo.meta, TestingSink(meta))
        return flow, (out, late, meta)

    flow, host = build(False)
    run_main(flow, gpu=False)
    flow, dev = build(False)
    run_main(flow, gpu=True)
    assert len(host[0]) > 1000 and len(host[1]) > 100
    assert dev[0] == host[0] and dev[2] == host[2]
    # the host's late stream carries the expanded item (ts_us, value), the device's the value (nothing for counts)
    assert [(k, w) for k, (w, _v) in dev[1]] == [(k, w) for k, (w, _v) in host[1]]
    if red != "count":
        assert [v for _k, (_w, v) in dev[1]] == [v[1] for _k, (_w, v) in host[1]]
    flow, cols = build(True)
    run_main(flow, gpu=True)
    assert all(isinstance(c, win.WindowColumns) for _k, c in cols[0]) and len(cols[0]) <= len(batches) + 1
    assert [r for _k, c in cols[0] for r in c.rows()] == host[0]
    assert [r for _k, c in cols[2] for r in c.rows()] == host[2]
