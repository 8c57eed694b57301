"""`collect_window` over session windows with the CUDA path enabled (run_main(..., gpu=True)): the engine hands collects
into list / set / dict over a `SessionWindower` to K12 (`bw_scwin_*`); the `down`, `late` and `meta` streams must equal
the host engine's, containers compared by their iteration order (``list(c)``, ``list(d.items())``).  -m gpu."""

import random
from datetime import datetime, timedelta, timezone

import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
import bytewax_b200.operators.windowing as win  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.operators.windowing import EventClock, SessionWindower, SystemClock  # noqa: E402
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


def _iter_order(rows):
    """Every row with each container replaced by its iteration order (dicts: their items)."""
    out = []
    for k, (w, c) in rows:
        if isinstance(c, dict):
            c = ("dict", list(c.items()))
        elif isinstance(c, (set, list)):
            c = (type(c).__name__, list(c))
        out.append((k, w, c))
    return out


@pytest.fixture
def k12_calls(monkeypatch):
    """The items of every device activation of a session collect step, to check that the CUDA path ran all of them."""
    calls = []
    orig = engine._GpuSessionCollectWindowStep.on_epoch

    def on_epoch(self, epoch, items):
        rows = orig(self, epoch, items)
        assert self.jwin is not None
        calls.append(len(items))
        return rows

    monkeypatch.setattr(engine._GpuSessionCollectWindowStep, "on_epoch", on_epoch)
    return calls


@pytest.fixture
def flat_differs(monkeypatch):
    """Counts the containers the step built whose flat replay of the same handles iterates differently: when it is
    positive, a step that rebuilt containers flat would have failed the comparison with the host engine."""
    n = [0]
    orig = engine._GpuSessionCollectWindowStep._session_container

    def session_container(self, handles, merges):
        c = orig(self, handles, merges)
        flat = self._container(handles)
        n[0] += (list(c.items()) if isinstance(c, dict) else list(c)) != (list(flat.items()) if isinstance(flat, dict) else list(flat))
        return c

    monkeypatch.setattr(engine._GpuSessionCollectWindowStep, "_session_container", session_container)
    return n


def _both(build):
    outs = []
    for gpu in (False, True):
        flow, sinks = build()
        run_main(flow, gpu=gpu)
        outs.append(sinks)
    return outs


def _items(seed, n=600, keys=12):
    rnd = random.Random(seed)
    out = []
    for i in range(n):
        t = ALIGN + timedelta(seconds=i // 8 + rnd.uniform(-6, 6))
        if rnd.random() < 0.05:
            t -= timedelta(seconds=rnd.uniform(10, 40))
        out.append((f"user{rnd.randrange(keys)}", t, i))
    return out


def _collect_flow(items, into, ordered, value, ts_of, gap=3 * S, wait=2 * S, clock=None):
    def make(keyed):
        c = clock or EventClock(ts_of, wait_for_system_duration=wait, now_getter=lambda: FROZEN)
        return win.collect_window("collect", op.map_value("val", keyed, value), c, SessionWindower(gap=gap), into=into, ordered=ordered)

    return _flow(items, make, batch_size=41)


@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("into", [list, set, dict])
def test_matches_host_engine(k12_calls, flat_differs, into, ordered):
    items = _items(3 + ordered)
    if into is dict:  # (key, (ts, i)): keys repeat, so merges overwrite
        value, ts_of = (lambda e: (e[2] % 5, (e[1], f"v{e[2]}"))), (lambda v: v[1][0])
    else:  # (ts, small int): small ints share a set's slots, so a merged set iterates unlike a flat replay
        value, ts_of = (lambda e: (e[1], (e[2] * 7919) % 61)), (lambda v: v[0])
    host, gpu = _both(lambda: _collect_flow(items, into, ordered, value, ts_of))
    assert host[0] and host[1]
    assert ordered or any(m.merged_ids for _k, (_w, m) in host[2])
    assert _iter_order(gpu[0]) == _iter_order(host[0])
    assert gpu[1] == host[1] and gpu[2] == host[2]
    assert sum(k12_calls) == len(items)  # every item went through a device activation
    if into is set and not ordered:
        assert flat_differs[0] > 0


def test_set_of_strings_matches_host_engine(k12_calls):
    items = _items(8)
    host, gpu = _both(lambda: _collect_flow(items, set, False, lambda e: (e[1], f"page{e[2] % 23}"), lambda v: v[0]))
    assert _iter_order(gpu[0]) == _iter_order(host[0]) and gpu[1:] == host[1:] and sum(k12_calls) == len(items)


def test_clickstream_sessions_per_user(k12_calls):
    """A search-log shaped flow: click events per user, sessionised with a 10 s gap (EventClock waiting 1 s), then a
    statistic per session -- the share of searches that led to a click."""
    rnd = random.Random(21)
    events = []
    for u in range(30):
        t = ALIGN + timedelta(seconds=rnd.uniform(0, 60))
        for _ in range(rnd.randint(3, 25)):
            t += timedelta(seconds=rnd.expovariate(1 / 6))
            events.append({"user": u, "type": rnd.choice(["search", "click", "click", "result"]), "time": t})
    rnd.shuffle(events)

    def build():
        down, meta = [], []
        flow = Dataflow("clicks")
        keyed = op.key_on("user", op.input("in", flow, TestingSource(events, batch_size=50)), lambda e: str(e["user"]))
        wo = win.collect_window("sessions", keyed, EventClock(lambda e: e["time"], wait_for_system_duration=S, now_getter=lambda: FROZEN),
                                SessionWindower(gap=10 * S))

        def ctr(wid_events):
            wid, evs = wid_events
            searches = sum(e["type"] == "search" for e in evs)
            clicks = sum(e["type"] == "click" for e in evs)
            return (wid, len(evs), clicks / searches if searches else None)

        op.output("out", op.map_value("ctr", wo.down, ctr), TestingSink(down))
        op.output("meta", wo.meta, TestingSink(meta))
        return flow, (down, meta)

    host, gpu = _both(build)
    assert host[0] and gpu == host and sum(k12_calls) == len(events)


def test_system_clock(k12_calls):
    items = [(f"k{i % 4}", None, i) for i in range(200)]
    host, gpu = _both(lambda: _collect_flow(items, list, False, lambda e: e[2], None, clock=SystemClock()))
    # (the sessions' bounds are the runs' own system times: only the lists are compared)
    assert [(k, (w, list(c))) for k, (w, c) in gpu[0]] == [(k, (w, list(c))) for k, (w, c) in host[0]] and sum(k12_calls) == len(items)


def test_fallback_unhashable_set_value_in_first_batch():
    items = [("a", ALIGN, 1), ("a", ALIGN + S, 2)]
    errs = []
    for gpu in (False, True):
        flow, _ = _collect_flow(items, set, False, lambda e: (e[1], [e[2]]), lambda v: v[0])
        with pytest.raises(Exception) as ei:
            run_main(flow, gpu=gpu)
        errs.append((type(ei.value), str(ei.value), repr(ei.value.__cause__)))
    assert errs[0] == errs[1] and "unhashable" in errs[0][2]  # the host logic raised in both runs


def test_fallback_non_pair_dict_value_in_first_batch():
    items = [("a", ALIGN, 1), ("a", ALIGN + S, 2)]
    msgs = []
    for gpu in (False, True):
        flow, _ = _collect_flow(items, dict, False, lambda e: 5, lambda v: ALIGN)
        with pytest.raises(Exception) as ei:
            run_main(flow, gpu=gpu)
        msgs.append(str(ei.value))
    assert msgs[0] == msgs[1]  # the host logic raised in both runs
