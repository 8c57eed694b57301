"""Session-window flows with the CUDA path enabled (run_main(..., gpu=True)): the recogniser hands count / reduce(add, max,
min) / max / min folds over a SessionWindower to K7 (`bw_session_*`); the `down`, `late` and `meta` streams (with the
merged session ids) must equal the host engine's.  -m gpu."""

import operator
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.operators.windowing import ZERO_TD, EventClock, SessionWindower  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)
S = timedelta(seconds=1)


class I(int):  # noqa: E742 - a number that carries its event time
    pass


class F(float):
    pass


def _num(cls, v, ts):
    x = cls(v)
    x.ts = ts
    return x


def _flow(items, windower_op, clock, batch_size=37, tick=None):
    down, late, meta = [], [], []
    flow = Dataflow("df")
    s = op.input("inp", flow, TestingSource(items, batch_size=batch_size))
    if tick is not None:
        s = op.map("tick", s, tick)
    wo = windower_op(s, clock)
    op.output("out", wo.down, TestingSink(down))
    op.output("late", wo.late, TestingSink(late))
    op.output("meta", wo.meta, TestingSink(meta))
    return flow, (down, late, meta)


def _both(build):
    outs = []
    for gpu in (False, True):
        flow, sinks = build()
        run_main(flow, gpu=gpu)
        outs.append(sinks)
    return outs


@pytest.fixture
def k7_steps(monkeypatch):
    """Records every session step that folded an activation on the device, to check that the CUDA path really ran."""
    made = []
    orig = engine._GpuSessionStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)  # (a fallback to the host raises before this returns)
        assert self.sess is not None
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuSessionStep, "on_epoch", on_epoch)
    return made


def test_count_window_reference_session_expectation(k7_steps):
    # pytests/operators/windowing/test_fold_window.py:97-140, counting instead of collecting
    secs = (1, 5, 11, 12, 13, 14, 20, 1)
    inp = [{"t": ALIGN + s * S, "v": c} for s, c in zip(secs, "abcdefgh")]

    def build():
        return _flow(inp, lambda s, clock: win.count_window("cnt", s, clock, SessionWindower(5 * S), lambda e: "ALL"),
                     EventClock(lambda e: e["t"], ZERO_TD, now_getter=lambda: FROZEN), batch_size=1)

    host, gpu = _both(build)
    assert host[0] == [("ALL", (0, 2)), ("ALL", (1, 4)), ("ALL", (2, 1))]
    assert host[1] == [("ALL", (-1, inp[-1]))]
    assert gpu == host and k7_steps


def _numeric_items(seed, n, cls, n_keys=25):
    rnd = np.random.default_rng(seed)
    items = []
    for i in range(n):
        ts = ALIGN + timedelta(seconds=float(i * 0.02 + rnd.uniform(-3, 3)))
        v = int(rnd.integers(-50, 50)) if cls is I else float(rnd.choice([0.1, 0.2, 0.3, 1e16, -1e16, -0.0, 0.0, 2.5]))
        items.append((f"user{int(rnd.integers(0, n_keys))}", _num(cls, v, ts)))  # string keys: interned on the device
    return items


@pytest.mark.parametrize("name,make,cls", [
    ("reduce_add_int", lambda s, c: win.reduce_window("r", s, c, SessionWindower(S // 2), operator.add), I),
    ("reduce_add_float", lambda s, c: win.reduce_window("r", s, c, SessionWindower(S // 2), operator.add), F),
    ("reduce_max", lambda s, c: win.reduce_window("r", s, c, SessionWindower(S // 3), max), F),
    ("reduce_min", lambda s, c: win.reduce_window("r", s, c, SessionWindower(S // 3), min), I),
    ("max_window", lambda s, c: win.max_window("m", s, c, SessionWindower(S // 4)), F),
    ("min_window", lambda s, c: win.min_window("m", s, c, SessionWindower(S)), I),
])
def test_numeric_session_folds_match_host(k7_steps, name, make, cls):
    items = _numeric_items(len(name), 4000, cls)

    def build():
        return _flow(items, make, EventClock(lambda v: v.ts, S, now_getter=lambda: FROZEN))

    host, gpu = _both(build)
    assert len(host[0]) > 100 and len(host[1]) > 10 and any(m.merged_ids for _k, (_w, m) in host[2])
    for h, g in zip(host, gpu):
        assert [(k, (w, float(v) if isinstance(v, float) else v)) for k, (w, v) in g] == \
               [(k, (w, float(v) if isinstance(v, float) else v)) for k, (w, v) in h]
    if cls is F:  # the bits of every float accumulator, signed zeros included
        bits = lambda rows: [np.float64(v).view(np.uint64) for _k, (_w, v) in rows]  # noqa: E731
        assert bits(gpu[0]) == bits(host[0])
    assert k7_steps


def test_count_window_stepping_clock_and_notify(k7_steps):
    """A moving `now_getter`: idle keys' sessions close in the notify phase, and drift makes items late."""
    now_box = [ALIGN]
    # (key, event time, system time of arrival)
    raw = [("a", 1.0, 2.0), ("a", 1.5, 2.0), ("b", 1.8, 2.5), ("c", 9.5, 9.6), ("c", 11.0, 10.0), ("z", 12.0, 13.0),
           ("z", 14.0, 15.0), ("a", 3.0, 16.0), ("c", 12.0, 16.5), ("z", 27.0, 27.5), ("b", 26.0, 28.0), ("b", 27.0, 28.5)]
    items = [(k, (ALIGN + ev * S, ALIGN + sy * S)) for k, ev, sy in raw]

    def tick(kv):
        now_box[0] = kv[1][1]
        return kv

    def build():
        now_box[0] = ALIGN
        clock = EventClock(lambda kv: kv[1][0], ZERO_TD, now_getter=lambda: now_box[0])
        return _flow(items, lambda s, c: win.count_window("cnt", s, c, SessionWindower(2 * S), lambda kv: kv[0]), clock,
                     batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[1] and host[0][0][0] in ("a", "b")
    assert gpu == host and k7_steps


def test_system_clock_sessions(monkeypatch, k7_steps):
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0), ("b", 2.0), ("a", 3.0), ("z", 12.0), ("a", 14.0), ("a", 15.0), ("z", 31.0), ("b", 33.0)]
    items = [(k, ALIGN + sy * S) for k, sy in raw]

    def tick(kv):
        now_box[0] = kv[1]
        return kv

    def build():
        now_box[0] = ALIGN
        return _flow(items, lambda s, c: win.count_window("cnt", s, c, SessionWindower(5 * S), lambda kv: kv[0]), win.SystemClock(),
                     batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[0][:2] == [("a", (0, 2)), ("b", (0, 1))]
    assert gpu == host and k7_steps


def test_non_numeric_values_fall_back_to_the_host(k7_steps):
    items = [("k", (ALIGN + i * S, s)) for i, s in enumerate(["x", "y", "z"])]

    def build():
        clock = EventClock(lambda v: v[0], ZERO_TD, now_getter=lambda: FROZEN)
        return _flow(items, lambda s, c: win.reduce_window("r", s, c, SessionWindower(5 * S), operator.add), clock)

    host, gpu = _both(build)
    assert host[0] == [("k", (0, (ALIGN, "x", ALIGN + S, "y", ALIGN + 2 * S, "z")))]
    assert gpu == host


def test_decimal_keys_keep_the_device_order(k7_steps):
    """Canonical decimal keys are not interned, so the engine passes the device's row order through unchanged: it must be
    ascending key TEXT across every digit-count boundary (src/operators.rs:758-767), as on the host."""
    names = ["0", "9", "10", "99", "100", "999", "1000", "9999999999", "10000000000", "9223372036854775807", "1", "2"]
    items = [(k, (ALIGN + (i % 3) * S, i)) for i, k in enumerate(names * 3)] + [(k, (ALIGN + 30 * S, 0)) for k in names]
    items += [(k, (ALIGN, -1)) for k in names[::-1]]  # late

    def build():
        clock = EventClock(lambda kv: kv[1][0], ZERO_TD, now_getter=lambda: FROZEN)
        return _flow(items, lambda s, c: win.count_window("cnt", s, c, SessionWindower(5 * S), lambda kv: kv[0]), clock,
                     batch_size=len(names) * 3)

    host, gpu = _both(build)
    first = [k for k, _ in host[0][: len(names)]]
    assert first == sorted(names) and first != sorted(names, key=int)
    assert len(host[1]) == len(names)
    assert gpu == host and k7_steps and not any(st.resort for st in k7_steps)
