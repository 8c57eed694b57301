"""`join_window` over session windows with the CUDA path enabled (run_main(..., gpu=True)): the recogniser hands first /
last session joins to K10 (`bw_sjwin_*`); the `down`, `late` and `meta` streams must equal the host engine's.  -m gpu."""

from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.operators.windowing import EventClock, SessionWindower  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)
S = timedelta(seconds=1)


def _flow(side_items, make, batch_size=37, tick=None):
    down, late, meta = [], [], []
    flow = Dataflow("df")
    sides = []
    for i, items in enumerate(side_items):
        s = op.input(f"in{i}", flow, TestingSource(items, batch_size=batch_size))
        if tick is not None:
            s = op.map(f"tick{i}", s, tick)
        sides.append(s)
    wo = make(sides)
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
def k10_steps(monkeypatch):
    """Records every session-join step that ran an activation on the device, to check that the CUDA path really ran."""
    made = []
    orig = engine._GpuSessionJoinWindowStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert self.jwin is not None
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuSessionJoinWindowStep, "on_epoch", on_epoch)
    return made


# pytests/operators/windowing/test_join_window.py: gap 10 s, wait forever, one key; values (ts, value)
REF_CASES = [("first", "complete", [(0, 1)], [(2, 3), (1, 2)], [(1, 2)]),
             ("last", "complete", [(0, 1)], [(1, 2)], [(1, 2)]),
             ("last", "final", [(0, 1)], [(1, 2), (2, 3)], [(1, 3)]),
             (None, None, [(0, 1)], [(1, 2), (2, 3)], [(1, 3)]),
             ("last", "running", [(0, 1)], [(1, 2), (2, 3)], [(1, None), (1, 2), (1, 3)])]


@pytest.mark.parametrize("case", range(len(REF_CASES)))
def test_reference_session_joins(k10_steps, case):
    ins, emit, left, right, want = REF_CASES[case]
    at = datetime(2024, 1, 1, tzinfo=timezone.utc)
    sides = [[("ALL", (at + t * S, v)) for t, v in left], [("ALL", (at + t * S, v)) for t, v in right]]

    def build():
        clock = EventClock(lambda x: x[0], wait_for_system_duration=timedelta.max)
        kw = {} if ins is None else dict(insert_mode=ins, emit_mode=emit)
        return _flow(sides, lambda s: win.join_window("join", clock, SessionWindower(10 * S), *s, **kw))

    host, gpu = _both(build)
    assert [tuple(None if v is None else v[1] for v in t) for _k, (_w, t) in gpu[0]] == want
    assert gpu == host and k10_steps


def _items(seed, n_sides, n=3000, n_keys=40, keys=None, step=0.01):
    rnd = np.random.default_rng(seed)
    out = [[] for _ in range(n_sides)]
    for i in range(n):
        ts = ALIGN + timedelta(seconds=float(i * step + rnd.uniform(-3, 3)))
        k = keys[int(rnd.integers(0, len(keys)))] if keys else f"user{int(rnd.integers(0, n_keys))}"
        out[int(rnd.integers(0, n_sides))].append((k, {"ts": ts, "i": i}))
    return out


MODES = [(i, e) for i in ("first", "last") for e in ("complete", "final", "running")]


@pytest.mark.parametrize("ins,emit", MODES)
@pytest.mark.parametrize("ordered", [True, False])
def test_modes_match_host(k10_steps, ins, emit, ordered):
    """Unordered flows merge sessions (their arrival order jumps back and forth), in first and last mode alike."""
    n_sides = 1 + (MODES.index((ins, emit)) + ordered) % 4
    items = _items(7 + MODES.index((ins, emit)), n_sides, step=0.05)

    def build():
        clock = EventClock(lambda v: v["ts"], 2 * S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, SessionWindower(S // 4), *s, insert_mode=ins, emit_mode=emit,
                                                      ordered=ordered))

    host, gpu = _both(build)
    assert gpu == host and k10_steps
    assert (len(host[0]) > 10 or emit == "complete") and len(host[1]) > 10 and len(host[2]) > 50
    if not ordered:
        assert any(m.merged_ids for _k, (_w, m) in host[2])


def test_decimal_keys_keep_the_device_order(k10_steps):
    names = ["0", "9", "10", "99", "100", "999", "1000", "9999999999", "10000000000", "9223372036854775807", "1", "2"]
    items = _items(3, 2, n=600, keys=names)

    def build():
        clock = EventClock(lambda v: v["ts"], timedelta(0), now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, SessionWindower(S // 10), *s, insert_mode="last", emit_mode="running",
                                                      ordered=False), batch_size=200)

    host, gpu = _both(build)
    assert len(host[1]) > 10 and gpu == host and k10_steps and not any(st.resort for st in k10_steps)


def test_stepping_clock_and_notify(k10_steps):
    """A moving `now_getter`: idle keys' sessions close (and ordered queues flush) in the notify phase."""
    now_box = [ALIGN]
    raw = [("a", 1.0, 2.0, 0), ("a", 1.5, 2.0, 1), ("b", 1.8, 2.5, 0), ("c", 9.5, 9.6, 1), ("c", 11.0, 10.0, 0), ("z", 12.0, 13.0, 1),
           ("z", 14.0, 15.0, 0), ("a", 3.0, 16.0, 1), ("c", 12.0, 16.5, 1), ("z", 27.0, 27.5, 0), ("b", 26.0, 28.0, 1), ("b", 27.0, 28.5, 0)]
    sides = [[(k, (ALIGN + ev * S, ALIGN + sy * S)) for k, ev, sy, sd in raw if sd == i] for i in range(2)]

    def tick(kv):
        now_box[0] = max(now_box[0], kv[1][1])
        return kv

    for ordered in (True, False):
        def build():
            now_box[0] = ALIGN
            clock = EventClock(lambda v: v[0], S, now_getter=lambda: now_box[0])
            return _flow(sides, lambda s: win.join_window("j", clock, SessionWindower(2 * S), *s, ordered=ordered), batch_size=1, tick=tick)

        host, gpu = _both(build)
        assert host[0] and gpu == host


def test_system_clock(monkeypatch, k10_steps):
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0, 0), ("b", 2.0, 1), ("a", 3.0, 1), ("z", 12.0, 0), ("a", 14.0, 0), ("a", 15.0, 1), ("z", 31.0, 1), ("b", 33.0, 0)]
    sides = [[(k, ALIGN + sy * S) for k, sy, sd in raw if sd == i] for i in range(2)]

    def tick(kv):
        now_box[0] = max(now_box[0], kv[1])
        return kv

    def build():
        now_box[0] = ALIGN
        return _flow(sides, lambda s: win.join_window("j", win.SystemClock(), SessionWindower(5 * S), *s, emit_mode="running"),
                     batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[0] and gpu == host and k10_steps
