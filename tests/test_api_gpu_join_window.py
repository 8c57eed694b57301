"""`join_window` flows with the CUDA path enabled (run_main(..., gpu=True)): the recogniser hands first / last joins over
tumbling and sliding windows to K8 (`bw_jwin_*`); the `down`, `late` and `meta` streams must equal the host engine's.
-m gpu."""

from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.operators.windowing import ZERO_TD, EventClock, SessionWindower, SlidingWindower, TumblingWindower  # noqa: E402
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
def k8_steps(monkeypatch):
    """Records every join-window step that ran an activation on the device, to check that the CUDA path really ran."""
    made = []
    orig = engine._GpuJoinWindowStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert self.jwin is not None
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuJoinWindowStep, "on_epoch", on_epoch)
    return made


def test_guide_walkthrough(k8_steps):
    # docs/guide/concepts/joins.md:470-634
    at = datetime(2023, 12, 14, tzinfo=timezone.utc)
    names = [("123", {"user_id": 123, "at": at, "name": "Bee"}), ("456", {"user_id": 456, "at": at, "name": "Hive"})]
    emails = [("123", {"user_id": 123, "at": at + timedelta(minutes=15), "email": "bee@bytewax.io"}),
              ("456", {"user_id": 456, "at": at + timedelta(hours=1, minutes=15), "email": "hive@bytewax.io"})]

    def build():
        clock = EventClock(ts_getter=lambda x: x["at"], wait_for_system_duration=timedelta(0), now_getter=lambda: FROZEN)
        windower = TumblingWindower(length=timedelta(hours=1), align_to=datetime(2023, 1, 1, tzinfo=timezone.utc))
        return _flow([names, emails], lambda s: win.join_window("join", clock, windower, *s))

    host, gpu = _both(build)
    assert [(k, w, tuple(v and (v.get("name") or v.get("email")) for v in t)) for k, (w, t) in host[0]] == [
        ("456", 8328, ("Hive", None)), ("123", 8328, ("Bee", "bee@bytewax.io")), ("456", 8329, (None, "hive@bytewax.io"))]
    assert gpu == host and k8_steps


def _items(seed, n_sides, n=3000, n_keys=40, keys=None):
    rnd = np.random.default_rng(seed)
    out = [[] for _ in range(n_sides)]
    for i in range(n):
        ts = ALIGN + timedelta(seconds=float(i * 0.01 + rnd.uniform(-3, 3)))
        k = keys[int(rnd.integers(0, len(keys)))] if keys else f"user{int(rnd.integers(0, n_keys))}"
        out[int(rnd.integers(0, n_sides))].append((k, {"ts": ts, "i": i}))
    return out


MODES = [(i, e) for i in ("first", "last") for e in ("complete", "final", "running")]


@pytest.mark.parametrize("ins,emit", MODES)
@pytest.mark.parametrize("ordered", [True, False])
def test_modes_match_host(k8_steps, ins, emit, ordered):
    n_sides = 1 + (MODES.index((ins, emit)) + ordered) % 4
    sliding = MODES.index((ins, emit)) % 2 == 0
    windower = SlidingWindower(3 * S, S, ALIGN + timedelta(milliseconds=250)) if sliding else TumblingWindower(2 * S, ALIGN)
    items = _items(7 + MODES.index((ins, emit)), n_sides)

    def build():
        clock = EventClock(lambda v: v["ts"], S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, windower, *s, insert_mode=ins, emit_mode=emit, ordered=ordered))

    host, gpu = _both(build)
    assert gpu == host and k8_steps
    assert len(host[0]) > 10 and len(host[1]) > 10 and len(host[2]) > 50


@pytest.mark.parametrize("n_sides", [1, 2, 3, 4])
def test_side_counts_match_host(k8_steps, n_sides):
    items = _items(50 + n_sides, n_sides, n=1500)

    def build():
        clock = EventClock(lambda v: v["ts"], 2 * S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, TumblingWindower(S, ALIGN), *s, insert_mode="first", emit_mode="final"))

    host, gpu = _both(build)
    assert len(host[0]) > 50 and gpu == host and k8_steps


def test_decimal_keys_keep_the_device_order(k8_steps):
    names = ["0", "9", "10", "99", "100", "999", "1000", "9999999999", "10000000000", "9223372036854775807", "1", "2"]
    items = _items(3, 2, n=600, keys=names)

    def build():
        clock = EventClock(lambda v: v["ts"], ZERO_TD, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.join_window("j", clock, TumblingWindower(S, ALIGN), *s, insert_mode="last", emit_mode="running"),
                     batch_size=200)

    host, gpu = _both(build)
    assert len(host[1]) > 10 and gpu == host and k8_steps and not any(st.resort for st in k8_steps)


def test_stepping_clock_and_notify(k8_steps):
    """A moving `now_getter`: idle keys' windows close (and ordered queues flush) in the notify phase."""
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
            return _flow(sides, lambda s: win.join_window("j", clock, TumblingWindower(2 * S, ALIGN), *s, ordered=ordered),
                         batch_size=1, tick=tick)

        host, gpu = _both(build)
        assert host[0] and gpu == host


def test_system_clock(monkeypatch, k8_steps):
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0, 0), ("b", 2.0, 1), ("a", 3.0, 1), ("z", 12.0, 0), ("a", 14.0, 0), ("a", 15.0, 1), ("z", 31.0, 1), ("b", 33.0, 0)]
    sides = [[(k, ALIGN + sy * S) for k, sy, sd in raw if sd == i] for i in range(2)]

    def tick(kv):
        now_box[0] = max(now_box[0], kv[1])
        return kv

    def build():
        now_box[0] = ALIGN
        return _flow(sides, lambda s: win.join_window("j", win.SystemClock(), TumblingWindower(5 * S, ALIGN), *s, emit_mode="running"),
                     batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[0] and gpu == host and k8_steps


@pytest.mark.parametrize("what", ["product", "session", "five_sides", "to_system_utc"])
def test_out_of_scope_stays_on_the_host(monkeypatch, what):
    made = []
    monkeypatch.setattr(engine, "_GpuJoinWindowStep", lambda *a: made.append(a) or pytest.fail("K8 step built"))
    n_sides = 5 if what == "five_sides" else 2
    items = _items(11, n_sides, n=400, n_keys=5)

    def build():
        kw = {"to_system_utc": lambda t: t} if what == "to_system_utc" else {}
        clock = EventClock(lambda v: v["ts"], S, now_getter=lambda: FROZEN, **kw)
        windower = SessionWindower(S) if what == "session" else TumblingWindower(S, ALIGN)
        mode = "product" if what == "product" else "last"
        return _flow(items, lambda s: win.join_window("j", clock, windower, *s, insert_mode=mode))

    host, gpu = _both(build)
    assert host[0] and gpu == host and not made
