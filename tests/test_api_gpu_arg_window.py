"""`max_window` / `min_window` with ``by=`` with the CUDA path enabled (run_main(..., gpu=True)): the operators hand the
step to K11 (`bw_argwin_*`) over tumbling, sliding and session windows; the `down`, `late` and `meta` streams must equal
the host engine's, item for item.  -m gpu."""

import math
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import gpu as gpu_mod  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.errors import BytewaxRuntimeError  # noqa: E402
from bytewax_b200.operators.windowing import EventClock, SessionWindower, SlidingWindower, TumblingWindower  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)
S = timedelta(seconds=1)
BY = lambda e: e["val"]  # noqa: E731


@pytest.fixture
def k11_calls(monkeypatch):
    """Counts the activations the device ran (`ArgWindow.apply`), to check that the CUDA path really ran."""
    calls = []
    orig = gpu_mod.ArgWindow.apply

    def apply(self, *a, **k):
        calls.append(len(a[0]))
        return orig(self, *a, **k)

    monkeypatch.setattr(gpu_mod.ArgWindow, "apply", apply)
    return calls


def _flow(items, make, batch_size=37, tick=None):
    down, late, meta = [], [], []
    flow = Dataflow("df")
    s = op.input("inp", flow, TestingSource(items, batch_size=batch_size))
    if tick is not None:
        s = op.map("tick", s, tick)
    s = op.key_on("key", s, lambda e: e["user"])
    wo = make(s)
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


# pytests/operators/windowing/test_max_min_window.py
REF_INP = [
    {"time": ALIGN, "user": "a", "val": 1},
    {"time": ALIGN + 4 * S, "user": "a", "val": 9},
    {"time": ALIGN + 8 * S, "user": "a", "val": 3},
    {"time": ALIGN + 12 * S, "user": "a", "val": 10},
    {"time": ALIGN + 13 * S, "user": "a", "val": 4},
]


@pytest.mark.parametrize("fn,want", [("max_window", [1, 3]), ("min_window", [0, 4])])
def test_reference_max_min_window(k11_calls, fn, want):
    def build():
        clock = EventClock(lambda e: e["time"], wait_for_system_duration=timedelta(0))
        return _flow(REF_INP, lambda s: getattr(win, fn)("add", s, clock, TumblingWindower(length=10 * S, align_to=ALIGN), by=BY))

    host, gpu = _both(build)
    assert gpu[0] == [("a", (i, REF_INP[j])) for i, j in enumerate(want)]
    assert gpu == host and k11_calls


def _items(seed, n=3000, n_keys=40, floats=False, step=0.01):
    rnd = np.random.default_rng(seed)
    out = []
    for i in range(n):
        ts = ALIGN + timedelta(seconds=float(i * step + rnd.uniform(-3, 3)))
        if floats:
            val = float(rnd.choice([math.nan, -0.0, 0.0, math.inf, -math.inf, 5e-324])) if rnd.random() < 0.1 else float(rnd.integers(-5, 5)) / 2
        else:
            val = int(rnd.integers(-5, 5))
        out.append({"user": f"user{int(rnd.integers(0, n_keys))}", "ts": ts, "val": val, "i": i})
    return out


WINDOWERS = {
    "tumbling": lambda: TumblingWindower(length=2 * S, align_to=ALIGN),
    "sliding": lambda: SlidingWindower(length=3 * S, offset=S, align_to=ALIGN),
    "session": lambda: SessionWindower(gap=S // 4),
}


@pytest.mark.parametrize("windower", sorted(WINDOWERS))
@pytest.mark.parametrize("fn", ["max_window", "min_window"])
@pytest.mark.parametrize("floats", [False, True])
def test_event_clock_matches_host(k11_calls, windower, fn, floats):
    """Items out of order by up to 3 s with a 1 s wait: late rows; sessions merge.  The same item objects go to both
    runs, so NaN by-values compare equal by identity."""
    items = _items(11 + sorted(WINDOWERS).index(windower) * 4 + floats * 2 + (fn == "min_window"), floats=floats)

    def build():
        clock = EventClock(lambda e: e["ts"], S, now_getter=lambda: FROZEN)
        return _flow(items, lambda s: getattr(win, fn)("m", s, clock, WINDOWERS[windower](), by=BY))

    host, gpu = _both(build)
    assert gpu == host and k11_calls
    assert len(host[0]) > 50 and len(host[1]) > 10 and len(host[2]) == len(host[0])
    if windower == "session":
        assert any(m.merged_ids for _k, (_w, m) in host[2])


@pytest.mark.parametrize("windower", sorted(WINDOWERS))
def test_stepping_clock_and_notify(k11_calls, windower):
    """A moving `now_getter`: idle keys' windows close in the notify phase."""
    now_box = [ALIGN]
    raw = [("a", 1.0, 2.0, 3), ("a", 1.5, 2.0, 5), ("b", 1.8, 2.5, 1), ("c", 9.5, 9.6, 2), ("c", 11.0, 10.0, 2), ("z", 12.0, 13.0, 7),
           ("z", 14.0, 15.0, 7), ("a", 3.0, 16.0, 9), ("c", 12.0, 16.5, 0), ("z", 27.0, 27.5, 1), ("b", 26.0, 28.0, 4), ("b", 27.0, 28.5, 4)]
    items = [{"user": k, "ts": ALIGN + ev * S, "sys": ALIGN + sy * S, "val": v} for k, ev, sy, v in raw]

    def tick(e):
        now_box[0] = max(now_box[0], e["sys"])
        return e

    def build():
        now_box[0] = ALIGN
        clock = EventClock(lambda e: e["ts"], S, now_getter=lambda: now_box[0])
        return _flow(items, lambda s: win.max_window("m", s, clock, WINDOWERS[windower](), by=BY), batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[0] and gpu == host and k11_calls


@pytest.mark.parametrize("windower", sorted(WINDOWERS))
def test_system_clock(monkeypatch, k11_calls, windower):
    now_box = [ALIGN]
    monkeypatch.setattr(win, "_get_system_utc", lambda: now_box[0])
    raw = [("a", 1.0, 4), ("b", 2.0, 1), ("a", 3.0, 4), ("z", 12.0, 0), ("a", 14.0, 8), ("a", 15.0, 9), ("z", 31.0, 1), ("b", 33.0, 0)]
    items = [{"user": k, "sys": ALIGN + sy * S, "val": v} for k, sy, v in raw]

    def tick(e):
        now_box[0] = max(now_box[0], e["sys"])
        return e

    def build():
        now_box[0] = ALIGN
        return _flow(items, lambda s: win.min_window("m", s, win.SystemClock(), WINDOWERS[windower](), by=BY), batch_size=1, tick=tick)

    host, gpu = _both(build)
    assert host[0] and gpu == host and k11_calls


@pytest.mark.parametrize("bad", ["x", True, 1 << 63, None])
def test_unfit_by_in_the_first_batch_runs_on_host(k11_calls, bad):
    """A by-value the device cannot compare in the first batch: the step runs on the host logic, which may still succeed
    (the reference only calls `by` to compare two items)."""
    items = [{"user": "a", "ts": ALIGN, "val": bad}, {"user": "b", "ts": ALIGN + S, "val": 3}, {"user": "b", "ts": ALIGN + 2 * S, "val": 4}]

    def build():
        clock = EventClock(lambda e: e["ts"], timedelta(0), now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.max_window("m", s, clock, TumblingWindower(length=10 * S, align_to=ALIGN), by=BY), batch_size=10)

    host, gpu = _both(build)
    assert gpu == host and not k11_calls and [v["val"] for _k, (_w, v) in host[0]] == [bad, 4]


def test_mixed_int_and_float_in_the_first_batch_runs_on_host(k11_calls):
    items = [{"user": "a", "ts": ALIGN, "val": 2**53 + 1}, {"user": "a", "ts": ALIGN + S, "val": float(2**53)}]

    def build():
        clock = EventClock(lambda e: e["ts"], timedelta(0), now_getter=lambda: FROZEN)
        return _flow(items, lambda s: win.max_window("m", s, clock, TumblingWindower(length=10 * S, align_to=ALIGN), by=BY))

    host, gpu = _both(build)
    assert gpu == host and not k11_calls and gpu[0][0][1][1] is items[0]


@pytest.mark.parametrize("bad", ["x", True, 1 << 63, 2.5, KeyError])
def test_unfit_by_after_the_first_batch_raises(k11_calls, bad):
    items = [{"user": "a", "ts": ALIGN, "val": 1}, {"user": "a", "ts": ALIGN + S, "val": 2}, {"user": "a", "ts": ALIGN + 2 * S}]
    if bad is not KeyError:
        items[2]["val"] = bad
    clock = EventClock(lambda e: e["ts"], timedelta(0), now_getter=lambda: FROZEN)
    flow, _ = _flow(items, lambda s: win.max_window("m", s, clock, TumblingWindower(length=10 * S, align_to=ALIGN), by=BY), batch_size=2)
    with pytest.raises(BytewaxRuntimeError) as ei:
        run_main(flow, gpu=True)
    cause = ei.value.__cause__
    assert isinstance(cause, TypeError) and "stateful_batch" in str(cause) and k11_calls
