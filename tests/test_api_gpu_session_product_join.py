"""`join_window(insert_mode="product")` over `SessionWindower` with the CUDA path enabled (run_main(..., gpu=True)): the
recogniser hands these joins to K16 (`bw_spjwin_*`); the `down`, `late` and `meta` streams (merged ids included) must
equal the host engine's.  -m gpu."""

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
def k16_steps(monkeypatch):
    """Records every session product join step that ran an activation on the device, to check that K16 really ran."""
    made = []
    orig = engine._GpuSessionProductJoinWindowStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert type(self) is engine._GpuSessionProductJoinWindowStep
        assert self.jwin is not None and type(self.jwin).__name__ == "SessionProductJoinWindow"
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuSessionProductJoinWindowStep, "on_epoch", on_epoch)
    return made


def _items(seed, n_sides, n=1200, n_keys=30):
    rnd = np.random.default_rng(seed)
    out = [[] for _ in range(n_sides)]
    for i in range(n):
        ts = ALIGN + timedelta(seconds=float(i * 0.02 + rnd.uniform(-2, 2)))
        out[int(rnd.integers(0, n_sides))].append((f"user{int(rnd.integers(0, n_keys))}", {"ts": ts, "i": i}))
    return out


def _merged(meta):
    return sum(len(m.merged_ids) for _k, (_w, m) in meta)


@pytest.mark.parametrize("emit", ["complete", "final", "running"])
@pytest.mark.parametrize("ordered", [True, False])
def test_modes_match_host(k16_steps, emit, ordered):
    i = ["complete", "final", "running"].index(emit)
    n_sides = 1 + (i + 2 * ordered) % 4
    items = _items(7 + i + 3 * ordered, n_sides, n=500 if emit == "running" else 1200)

    def build():
        clock = EventClock(lambda v: v["ts"], S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, SessionWindower(S / 4), *s, insert_mode="product", emit_mode=emit,
                                                      ordered=ordered))

    host, gpu = _both(build)
    assert gpu == host and k16_steps
    assert host[0] and len(host[1]) > 5 and len(host[2]) > 20
    assert (_merged(host[2]) > 0) == (not ordered)  # unordered streams merge sessions; ordered ones never do


@pytest.mark.parametrize("n_sides", [1, 2, 3, 4])
def test_side_counts_match_host(k16_steps, n_sides):
    items = _items(50 + n_sides, n_sides, n=800)

    def build():
        clock = EventClock(lambda v: v["ts"], 2 * S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, SessionWindower(S / 5), *s, insert_mode="product", ordered=False))

    host, gpu = _both(build)
    assert len(host[0]) > 50 and gpu == host and k16_steps
    assert _merged(host[2]) > 0


def test_stepping_clock_and_notify(k16_steps):
    now_box = [ALIGN]
    raw = [("a", 1.0, 2.0, 0), ("a", 1.5, 2.0, 1), ("a", 1.7, 2.1, 1), ("b", 1.8, 2.5, 0), ("c", 9.5, 9.6, 1), ("c", 11.0, 10.0, 0),
           ("z", 12.0, 13.0, 1), ("z", 14.0, 15.0, 0), ("a", 3.0, 16.0, 1), ("c", 12.0, 16.5, 1), ("z", 27.0, 27.5, 0),
           ("b", 26.0, 28.0, 1), ("b", 27.0, 28.5, 0), ("b", 27.5, 28.6, 0), ("z", 13.0, 28.7, 1)]
    sides = [[(k, (ALIGN + ev * S, ALIGN + sy * S)) for k, ev, sy, sd in raw if sd == i] for i in range(2)]

    def tick(kv):
        now_box[0] = max(now_box[0], kv[1][1])
        return kv

    for ordered in (True, False):
        for emit in ("final", "running", "complete"):
            def build():
                now_box[0] = ALIGN
                clock = EventClock(lambda v: v[0], 3 * S, now_getter=lambda: now_box[0])
                return _flow(sides, lambda s: win.join_window("j", clock, SessionWindower(2 * S), *s, insert_mode="product",
                                                              emit_mode=emit, ordered=ordered), batch_size=1, tick=tick)

            host, gpu = _both(build)
            assert host[2] and gpu == host
    assert k16_steps


def test_system_clock(monkeypatch, k16_steps):
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0, 0), ("b", 2.0, 1), ("a", 3.0, 1), ("a", 3.5, 1), ("z", 12.0, 0), ("a", 14.0, 0), ("a", 15.0, 1), ("z", 31.0, 1),
           ("b", 33.0, 0)]
    sides = [[(k, ALIGN + sy * S) for k, sy, sd in raw if sd == i] for i in range(2)]

    def tick(kv):
        now_box[0] = max(now_box[0], kv[1])
        return kv

    def build():
        now_box[0] = ALIGN
        return _flow(sides, lambda s: win.join_window("j", win.SystemClock(), SessionWindower(5 * S), *s, insert_mode="product",
                                                      emit_mode="running"), batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[0] and gpu == host and k16_steps


@pytest.mark.parametrize("emit", ["complete", "final", "running"])
def test_two_workers(k16_steps, emit):
    """Two workers shard the keys and interleave their rows: each key's rows, in order, are the host engine's."""
    items = _items(90, 3, n=900 if emit != "running" else 450)

    def build():
        clock = EventClock(lambda v: v["ts"], S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, SessionWindower(S / 4), *s, insert_mode="product", emit_mode=emit,
                                                      ordered=False))

    flow, host = build()
    run_main(flow)
    flow, gpu = build()
    engine._Run(flow, 2, None, True).run()
    per_key = lambda rows: {k: [v for kk, v in rows if kk == k] for k, _ in rows}  # noqa: E731
    for h, g in zip(host, gpu):
        assert per_key(g) == per_key(h) and len(g) == len(h)
    assert host[0] and k16_steps


def test_other_calls_stay_off_k16():
    """More than 4 sides and a custom `to_system_utc` stay on the host engine; first / last over sessions stay on K10."""
    flow = Dataflow("df")
    ins = [op.input(f"in{i}", flow, TestingSource([])) for i in range(5)]
    clock = EventClock(lambda v: v, S)
    custom = EventClock(lambda v: v, S, to_system_utc=lambda t: t)
    assert win._session_product_join_window_plan(clock, SessionWindower(S), 5, "product", "final", True) is None
    assert win._session_product_join_window_plan(custom, SessionWindower(S), 2, "product", "final", True) is None
    p = win._join_window_plan(clock, SessionWindower(S), 2, "last", "final", True)
    assert type(engine._gpu_step_for("j", p)) is engine._GpuSessionJoinWindowStep
    assert ins
