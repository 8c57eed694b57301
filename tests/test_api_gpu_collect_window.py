"""`collect_window` flows with the CUDA path enabled (run_main(..., gpu=True)): the recogniser hands collects into
list / set / dict over tumbling and sliding windows to K9 (`bw_collect_*`); the `down`, `late` and `meta` streams must
equal the host engine's.  -m gpu."""

from datetime import datetime, timedelta, timezone

import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.operators.windowing import EventClock, SlidingWindower, TumblingWindower  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)
S = timedelta(seconds=1)


def _flow(items, make, batch_size=37, key=lambda x: x[0]):
    down, late, meta = [], [], []
    flow = Dataflow("df")
    keyed = op.key_on("key", op.input("in", flow, TestingSource(items, batch_size=batch_size)), key)
    wo = make(keyed)
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
def k9_steps(monkeypatch):
    """Records every collect-window step that ran an activation on the device, to check that the CUDA path really ran."""
    made = []
    orig = engine._GpuCollectWindowStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert self.jwin is not None
        made.append(self)
        return rows

    monkeypatch.setattr(engine._GpuCollectWindowStep, "on_epoch", on_epoch)
    return made


def test_reference_collect_window_flow(k9_steps):
    # pytests/operators/windowing/test_collect_window.py
    inp = [(ALIGN, 1), (ALIGN + 8 * S, 3), (ALIGN + 4 * S, 2), (ALIGN + 13 * S, 5), (ALIGN + 12 * S, 4)]

    def build():
        clock = EventClock(lambda e: e[0], wait_for_system_duration=timedelta.max)
        windower = TumblingWindower(length=10 * S, align_to=ALIGN)
        return _flow(inp, lambda k: win.collect_window("collect_window", k, clock, windower), batch_size=1, key=lambda _e: "ALL")

    host, gpu = _both(build)
    assert [(w, [e[1] for e in vs]) for _k, (w, vs) in host[0]] == [(0, [1, 2, 3]), (1, [4, 5])]
    assert gpu == host and k9_steps


def test_docstring_example(k9_steps):
    # the operator's docstring (windowing.py:1436-1576)
    a = datetime(2023, 1, 1, tzinfo=timezone.utc)
    inp = [("a", a + 1 * S, 1), ("b", a + 2 * S, 2), ("a", a + 5 * S, 3), ("a", a + 11 * S, 4), ("b", a + 15 * S, 5)]

    def build():
        clock = EventClock(lambda e: e[1], wait_for_system_duration=timedelta(0), now_getter=lambda: FROZEN)
        windower = TumblingWindower(length=10 * S, align_to=a)
        return _flow(inp, lambda k: win.collect_window("collect", k, clock, windower))

    host, gpu = _both(build)
    assert len(host[0]) == 4 and gpu == host and k9_steps


def test_event_time_processing_shape(k9_steps):
    # examples/event_time_processing.py: tumbling, wait 10 s, out-of-order sensor readings
    import random

    rnd = random.Random(4)
    inp = [(f"sensor_{rnd.randrange(5)}", ALIGN + timedelta(milliseconds=rnd.randrange(0, 120_000)), i) for i in range(3000)]

    def build():
        clock = EventClock(lambda e: e[1], wait_for_system_duration=10 * S, now_getter=lambda: FROZEN)
        windower = TumblingWindower(length=5 * S, align_to=ALIGN)
        return _flow(inp, lambda k: win.collect_window("collect", k, clock, windower), batch_size=100)

    host, gpu = _both(build)
    assert host[1] and gpu == host and k9_steps


@pytest.mark.parametrize("into", [list, set, dict])
@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("shape", ["tumbling", "sliding"])
def test_into_order_shape(k9_steps, into, ordered, shape):
    import random

    rnd = random.Random(hash((into.__name__, ordered, shape)) & 0xFFFF)
    # (key, ts, value); the value is what is collected: (k, v) pairs for dict, with repeated ks so later values win
    inp = [(str(rnd.randrange(40)), ALIGN + timedelta(milliseconds=rnd.randrange(0, 200_000)), (rnd.randrange(8), i)) for i in range(4000)]

    def build():
        clock = EventClock(lambda e: e[1], wait_for_system_duration=3 * S, now_getter=lambda: FROZEN)
        windower = (TumblingWindower(length=10 * S, align_to=ALIGN) if shape == "tumbling"
                    else SlidingWindower(length=60 * S, offset=10 * S, align_to=ALIGN + timedelta(milliseconds=1234)))
        mapped = lambda k: op.map_value("v", k, lambda e: e[2] if into is dict else e)  # noqa: E731
        return _flow(inp, lambda k: win.collect_window("collect", mapped(k), _Clock(clock, into), windower, into=into, ordered=ordered))

    host, gpu = _both(build)
    assert host[0] and gpu == host and k9_steps
    if into is not list:
        assert all(type(v) is into for _k, (_w, v) in gpu[0])
        assert [list(v) if into is set else list(v.items()) for _k, (_w, v) in gpu[0]] == \
               [list(v) if into is set else list(v.items()) for _k, (_w, v) in host[0]]


def _Clock(clock, into):
    # dict values are (k, i) pairs: the timestamp travels in i
    if into is not dict:
        return clock
    return EventClock(lambda kv: ALIGN + timedelta(milliseconds=(kv[1] * 7919) % 200_000), clock.wait_for_system_duration, clock.now_getter)


def test_system_clock(monkeypatch, k9_steps):
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0), ("b", 2.0), ("a", 3.0), ("z", 12.0), ("a", 14.0), ("a", 15.0), ("z", 31.0), ("b", 33.0)]
    inp = [(k, ALIGN + sy * S) for k, sy in raw]

    def tick(kv):
        now_box[0] = max(now_box[0], kv[1][1])
        return kv

    def build():
        now_box[0] = ALIGN
        return _flow(inp, lambda k: win.collect_window("collect", op.map("tick", k, tick), win.SystemClock(), TumblingWindower(5 * S, ALIGN)),
                     batch_size=1)

    host, gpu = _both(build)
    assert host[0] and gpu == host and k9_steps


def test_string_keys_resorted(k9_steps):
    inp = [(k, ALIGN + timedelta(seconds=i % 50), i) for i, k in enumerate(["b", "a10", "a9", "Z", "é", "10", "9", "0x"] * 60)]

    def build():
        clock = EventClock(lambda e: e[1], wait_for_system_duration=2 * S, now_getter=lambda: FROZEN)
        return _flow(inp, lambda k: win.collect_window("collect", k, clock, TumblingWindower(length=5 * S, align_to=ALIGN)))

    host, gpu = _both(build)
    assert host[0] and gpu == host and k9_steps
    assert any(s.resort for s in k9_steps)


def test_dict_needs_pairs():
    """A non-pair value in the first batch sends the step to the host logic (`_GpuPlanUnfit`), which raises its own
    error; later, the device step raises the reference's message at ingest."""
    clock = EventClock(lambda e: ALIGN, wait_for_system_duration=timedelta.max)
    plan = win.GpuCollectWindowPlan(dict, True, clock, TumblingWindower(length=10 * S, align_to=ALIGN), "df.collect")
    step = engine._GpuCollectWindowStep("df.collect.fold_window.window.stateful_batch", plan)
    try:
        with pytest.raises(engine._GpuPlanUnfit):
            step.on_epoch(1, [("a", 5)])
        assert step.on_epoch(1, [("a", (1, 2)), ("b", ("x", [3]))]) == []
        with pytest.raises(TypeError, match="step 'df.collect' collecting into a `dict` requires `\\(key, value\\)` 2-tuple"):
            step.on_epoch(2, [("a", 5)])
        with pytest.raises(TypeError, match="collecting into a `dict`"):
            step.on_epoch(2, [("a", ([1], 2))])  # unhashable key: `d[k] = v` raises TypeError in the reference's folder too
    finally:
        step.release()
