"""Window folds with the CUDA path under a stepping `now_getter` (run_main(..., gpu=True)) against the host engine.
-m gpu.

Event time stays behind the getter here.  The host engine schedules its notify phases against the wall clock
(engine.py, like the reference's `Utc::now()` in src/operators.rs:674,808-812) and the GPU steps against the getter;
the two agree only while no key's watermark -- computed from the getter -- passes the getter's own now.  A getter that
is not the wall clock is a limit of the device path (DESIGN §10)."""

import operator
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.inputs import KeyedColumns  # noqa: E402
from bytewax_b200.operators.windowing import EventClock, SlidingWindower, TumblingWindower  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
A_US = 1_640_995_200_000_000
S = timedelta(seconds=1)


class I(int):  # noqa: E742 - a number that carries its event time and the system time it arrives at
    pass


@pytest.fixture
def device_steps(monkeypatch):
    """Every window step that folded an activation on the device."""
    made = []
    orig = engine._GpuWindowStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert self.fold is not None
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuWindowStep, "on_epoch", on_epoch)
    return made


def _items(seed, n=3000, n_keys=40):
    """System time steps 50 ms per item (about 600 distinct getter values over the batches); event time 0.5 .. 4 s
    behind it; a third of the keys go idle for 20 s stretches, so their windows close in notify phases."""
    rnd = np.random.default_rng(seed)
    out, sys_t = [], 0.0
    for i in range(n):
        sys_t += 0.05
        k = int(rnd.integers(0, n_keys))
        if k % 3 == 0 and int(sys_t) % 40 >= 20:
            k += 1
        v = I(int(rnd.integers(-50, 50)))
        v.ts = ALIGN + timedelta(seconds=sys_t - float(rnd.uniform(0.5, 4.0)))
        v.sys = ALIGN + timedelta(seconds=sys_t)
        out.append((f"k{k}", v))
    return out


def _flow(items, make, now_box, batch_size=23):
    down, late, meta = [], [], []
    flow = Dataflow("df")
    s = op.input("inp", flow, TestingSource(items, batch_size=batch_size))

    def tick(kv):
        now_box[0] = kv[1].sys
        return kv

    s = op.map("tick", s, tick)
    ts_of = lambda x: x[1].ts if isinstance(x, tuple) else x.ts  # noqa: E731  (count_window sees the (key, value) item)
    wo = make(s, EventClock(ts_of, 2 * S, now_getter=lambda: now_box[0]))
    op.output("out", wo.down, TestingSink(down))
    op.output("late", wo.late, TestingSink(late))
    op.output("meta", wo.meta, TestingSink(meta))
    return flow, (down, late, meta)


MAKERS = {
    "count_window": lambda s, c: win.count_window("c", s, c, TumblingWindower(3 * S, ALIGN), lambda kv: kv[0]),
    "reduce_add": lambda s, c: win.reduce_window("r", s, c, SlidingWindower(4 * S, 2 * S, ALIGN), operator.add),
    "reduce_max": lambda s, c: win.reduce_window("r", s, c, TumblingWindower(3 * S, ALIGN), max),
    "reduce_min": lambda s, c: win.reduce_window("r", s, c, SlidingWindower(5 * S, 2 * S, ALIGN), min),
    "max_window": lambda s, c: win.max_window("m", s, c, TumblingWindower(2 * S, ALIGN)),
    "min_window": lambda s, c: win.min_window("m", s, c, SlidingWindower(6 * S, 3 * S, ALIGN)),
}


@pytest.mark.parametrize("name", sorted(MAKERS))
def test_stepping_clock_matches_host(device_steps, name):
    items = _items(len(name))
    outs = []
    for gpu in (False, True):
        now_box = [ALIGN]
        flow, sinks = _flow(items, MAKERS[name], now_box)
        run_main(flow, gpu=gpu)
        outs.append(sinks)
    host, dev = outs
    assert len(host[0]) > 200 and host[1]
    assert [(k, (w, int(v))) for k, (w, v) in dev[0]] == [(k, (w, int(v))) for k, (w, v) in host[0]]
    assert [(k, w) for k, (w, _v) in dev[1]] == [(k, w) for k, (w, _v) in host[1]]
    assert dev[2] == host[2]
    assert device_steps


@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("red", ["count", "sum", "max"])
def test_fold_columns_stepping_clock(device_steps, red, ordered):
    """`fold_columns` batches under a getter that steps 100 ms per batch, event time 1 .. 3 s behind it, a third of
    the keys idle in every other 10 s: the ordered and unordered folds equal the host engine's."""
    rnd = np.random.default_rng(5 + ordered)
    batches, times = [], []
    for b in range(300):
        now = A_US + b * 100_000
        n = 200
        keys = rnd.integers(0, 90, n).astype(np.uint64)
        if (b // 100) % 2:
            keys[keys % np.uint64(3) == 0] += np.uint64(1)
        ts = now - rnd.integers(1_000_000, 3_000_000, n)
        batches.append(KeyedColumns(keys=keys, ts_us=ts.astype(np.int64),
                                    vals=None if red == "count" else rnd.integers(-50, 50, n).astype(np.int64)))
        times.append(ALIGN + timedelta(microseconds=now - A_US))

    def build():
        box, it = [ALIGN], iter(times)
        out, late, meta = [], [], []
        flow = Dataflow("df")
        s = op.input("inp", flow, TestingSource(batches))

        def tick(cols):
            box[0] = next(it)
            return cols

        s = op.map("tick", s, tick)
        wo = win.fold_columns("fold", s, red, TumblingWindower(S, ALIGN), S, ordered=ordered, now_getter=lambda: box[0])
        op.output("out", wo.down, TestingSink(out))
        op.output("late", wo.late, TestingSink(late))
        op.output("meta", wo.meta, TestingSink(meta))
        return flow, (out, late, meta)

    flow, host = build()
    run_main(flow, gpu=False)
    flow, dev = build()
    run_main(flow, gpu=True)
    assert len(host[0]) > 1000 and host[1]
    assert dev[0] == host[0] and dev[2] == host[2]
    assert [(k, w) for k, (w, _v) in dev[1]] == [(k, w) for k, (w, _v) in host[1]]
    assert device_steps


def test_custom_to_system_utc_runs_on_the_host(device_steps):
    """`to_system_utc` shifting close times by 30 s: the fold stays on the host engine, with the host's rows."""
    items = _items(3, n=600)
    outs = []
    for gpu in (False, True):
        now_box = [ALIGN]
        down = []
        flow = Dataflow("df")
        s = op.input("inp", flow, TestingSource(items, batch_size=23))
        s = op.map("tick", s, lambda kv: (now_box.__setitem__(0, kv[1].sys), kv)[1])
        clock = EventClock(lambda kv: kv[1].ts, 2 * S, now_getter=lambda: now_box[0], to_system_utc=lambda t: t + 30 * S)
        wo = win.count_window("c", s, clock, TumblingWindower(3 * S, ALIGN), lambda kv: kv[0])
        op.output("out", wo.down, TestingSink(down))
        run_main(flow, gpu=gpu)
        outs.append(down)
    assert outs[1] == outs[0] and len(outs[0]) > 50
    assert not device_steps


def test_ordered_fold_with_event_time_ahead_raises(device_steps):
    """An ordered fold whose event time leads the getter by more than the wait: the device cannot know the reference's
    queue head, refuses the notify phase, and the run stops with a TypeError naming the step."""
    batches, times = [], []
    for b in range(40):
        now = A_US + b * 500_000
        keys = np.arange(20, dtype=np.uint64) if b == 0 else np.array([100], np.uint64)  # (keys 0 .. 19 then idle)
        batches.append(KeyedColumns(keys=keys, ts_us=np.full(len(keys), now + 30_000_000 + b, np.int64), vals=None))
        times.append(ALIGN + timedelta(microseconds=now - A_US))

    box, it = [ALIGN], iter(times)
    flow = Dataflow("df")
    s = op.input("inp", flow, TestingSource(batches))
    s = op.map("tick", s, lambda cols: (box.__setitem__(0, next(it)), cols)[1])
    wo = win.fold_columns("fold", s, "count", TumblingWindower(S, ALIGN), 2 * S, ordered=True, now_getter=lambda: box[0])
    op.output("out", wo.down, TestingSink([]))
    with pytest.raises(Exception) as e:
        run_main(flow, gpu=True)
    err = e.value
    while err is not None and not isinstance(err, TypeError):
        err = err.__cause__ or err.__context__
    assert err is not None and "event time ahead of the system clock" in str(err) and "fold" in str(err)
