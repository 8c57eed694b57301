"""CPU restatement of `collect_window` into list / set / dict over session windows, on integer microseconds and value
HANDLES.  TEST INFRASTRUCTURE ONLY.

What the CUDA session collect (``bw_scwin``, csrc/bw_scwin.cuh) replaces (paths relative to the bytewax v0.21.1 tree):

* ``collect_window``       -> pysrc/bytewax/operators/windowing.py:1436-1576, callbacks :1356-1384
* ``_FoldWindowLogic``     -> windowing.py:1692-1714 (``on_merge``: ``state = merger(state, original.state)``)
* ``_WindowLogic``         -> windowing.py:1046-1190 (late test, queue, ordered flush, inserts, merges, close, notify_at)
* ``SessionWindower``      -> windowing.py:671-810 (``tests.session_oracle.SessionWindower``); never discarded
* ``EventClock``           -> windowing.py:230-310 (``oracle.pyoracle.EventClock``)
* engine                   -> src/operators.rs:755-806, :808-858 (notify), :862-894 (EOF)

A session's state here is what the device keeps: its handles in FLATTENED play order and its merge intervals, each block
``[start, end)`` of the list that one merged-away session (transitively) contributed, by start ascending then end
descending.  ``container`` rebuilds the reference's container from them with the reference's own calls.  Rows are
``[key, window_id, tag, payload]``: ``E`` ``[handles, intervals]``, ``L`` the handle (window -1), ``M`` ``[open_us,
close_us, sorted merged ids]``.  ``run_session_collect`` also reports the handles each call releases
(``bw_scwin_rows.released``).  Streams reuse the shape of ``tests/session_join_oracle.py``, one side.
"""

from __future__ import annotations

from datetime import timedelta
from typing import Dict, List, Optional

from oracle.pyoracle import UTC_MAX_US, UTC_MIN_US, EventClock, key_str
from tests import session_join_oracle as sj
from tests.session_oracle import LATE_SESSION_ID, SessionWindower

WAIT_FOREVER, S, A = sj.WAIT_FOREVER, sj.S, sj.A
INTOS = ("list", "set", "dict")


def dict_value(h: int):
    """The ``(key, value)`` pair a dict case carries for handle ``h``: keys repeat every 3 handles, so merges overwrite."""
    return (h % 3, h)


def _fold(into: str, state, v):
    if into == "list":
        state.append(v)
    elif into == "set":
        state.add(v)
    else:
        k, x = v
        state[k] = x
    return state


def _merge(into: str, a, b):
    if into == "list":
        return list.__add__(a, b)
    if into == "set":
        return set.union(a, b)
    a.update(b)  # _collect_dict_merger
    return a


def container(into: str, handles: List[int], intervals, value_of=lambda h: h):
    """The reference's container of one session: the folder per value, and at each interval the block's container built
    the same way, joined with the merger."""
    iv = [tuple(x) for x in intervals]

    def build(lo, hi, k):
        state = {"list": list, "set": set, "dict": dict}[into]()
        i = lo
        while i < hi:
            if k < len(iv) and iv[k][0] == i:
                end = iv[k][1]
                child, k = build(i, end, k + 1)
                state = _merge(into, state, child)
                i = end
                continue
            state = _fold(into, state, value_of(handles[i]))
            i += 1
        return state, k

    return build(0, len(handles), 0)[0]


def flat(into: str, handles: List[int], value_of=lambda h: h):
    """The container a flat replay of the handles gives (what sets must NOT be built by)."""
    return container(into, handles, [], value_of)


class SessionCollectLogic:
    """``_WindowLogic`` over a session windower and the collect fold per session, for one key."""

    def __init__(self, spec: dict, now_us: int):
        self.ordered = spec["ordered"]
        self.clock = EventClock(spec["wait_us"], now_us)
        self.windower = SessionWindower(spec["gap_us"])
        self.states: Dict[int, list] = {}  # session id -> [handles, intervals]
        self.queue: List[tuple] = []  # (handle, ts)
        self.last_watermark = UTC_MIN_US
        self.merges = 0

    def _flush(self, watermark: int) -> List[list]:
        # windowing.py:1095-1108
        if self.ordered:
            due = [e for e in self.queue if e[1] <= watermark]
            self.queue = [e for e in self.queue if not (e[1] <= watermark)]
            due.sort(key=lambda e: e[1])  # stable
        else:
            due, self.queue = self.queue, []
        for h, ts in due:  # _handle_inserts: the folder on the session open_for returned
            self.states.setdefault(self.windower.open_for(ts), [[], []])[0].append(h)
        for orig, into in self.windower.merged():  # _handle_merged: into.state = merger(into.state, orig.state)
            self.merges += 1
            a, b = self.states[into], self.states.pop(orig)
            base = len(a[0])
            a[1].append((base, base + len(b[0])))
            a[1].extend((s + base, e + base) for s, e in b[1])
            a[0].extend(b[0])
        events = []
        for wid, meta in self.windower.close_for(watermark):  # _handle_closed
            hs, iv = self.states.pop(wid)
            events.append([wid, "E", [hs, [list(x) for x in sorted(iv, key=lambda x: (x[0], -x[1]))]]])
            events.append([wid, "M", [meta[0], meta[1], sorted(meta[2])]])
        return events

    def on_batch(self, items) -> List[list]:
        """``items``: ``(handle, ts_us)`` in arrival order (windowing.py:1115-1133)."""
        self.clock.before_batch()
        events = []
        watermark = self.last_watermark
        for h, ts in items:
            _, watermark = self.clock.on_item(ts)
            self.last_watermark = watermark
            if ts < watermark:
                events.append([LATE_SESSION_ID, "L", h])
            else:
                self.queue.append((h, ts))
        return events + self._flush(watermark)

    def on_notify(self) -> List[list]:
        watermark = self.clock.on_notify()
        self.last_watermark = watermark
        return self._flush(watermark)

    def on_eof(self) -> List[list]:
        self.last_watermark = UTC_MAX_US
        return self._flush(UTC_MAX_US)

    def notify_at(self) -> Optional[int]:
        at = self.windower.notify_at()
        if self.ordered and self.queue:
            q = self.queue[0][1]
            at = q if at is None else min(at, q)
        return at

    def held(self) -> set:
        out = {h for st in self.states.values() for h in st[0]}
        out.update(e[0] for e in self.queue)
        return out


def run_session_collect(spec: dict, steps, eof: bool = True, stats: Optional[dict] = None):
    """``spec``: ordered, gap_us, wait_us.  ``steps``: ``["batch", now_us, keys, ts, values]`` or ``["notify", now_us]``;
    values are distinct ints (the handles).  ``stats`` gets ``merges``.  Returns ``(acts, released)``: the rows of every
    step (then EOF), and per step the sorted handles it released."""
    logics: Dict[str, SessionCollectLogic] = {}
    ids: Dict[str, int] = {}
    acts, released = [], []
    held: set = set()

    def settle(rows, incoming):
        nonlocal held
        now_held = set().union(*(lg.held() for lg in logics.values())) if logics else set()
        released.append(sorted((held | incoming) - now_held))
        held = now_held
        acts.append(rows)

    for step in steps:
        now = step[1]
        for lg in logics.values():
            lg.clock.now_us = now
        rows, incoming = [], set()
        if step[0] == "batch":
            grouped: Dict[str, list] = {}
            for k, t, v in zip(step[2], step[3], step[4]):
                ks = key_str(k)
                ids[ks] = int(k)
                grouped.setdefault(ks, []).append((v, int(t)))
                incoming.add(v)
            for ks in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
                lg = logics.get(ks)
                if lg is None:
                    lg = logics[ks] = SessionCollectLogic(spec, now)
                rows.extend([ids[ks], w, tag, p] for w, tag, p in lg.on_batch(grouped[ks]))
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now:
                    rows.extend([ids[ks], w, tag, p] for w, tag, p in logics[ks].on_notify())
        settle(rows, incoming)
    if eof:
        rows = []
        for ks in sorted(logics):
            rows.extend([ids[ks], w, tag, p] for w, tag, p in logics[ks].on_eof())
        settle(rows, set())
    if stats is not None:
        stats["merges"] = sum(lg.merges for lg in logics.values())
    return acts, released


def seeded_steps(seed: int, n_steps: int = 30, n_keys: int = 6, moving: bool = True):
    """K10's seeded streams (``tests/session_join_oracle.seeded_steps``) with the side column dropped; the spec keeps
    its order, gap and wait."""
    spec, steps = sj.seeded_steps(seed, n_steps, n_keys, moving)
    spec = dict(ordered=spec["ordered"], gap_us=spec["gap_us"], wait_us=spec["wait_us"])
    return spec, [s if s[0] == "notify" else s[:4] + [s[5]] for s in steps]


SEEDED = range(48)


# ---- golden rows: what the reference's own logic returns, with the containers as JSON ---------------------------------
# A case's values are the reference's items: into=list carries the handle itself, into=set `set_value(h)` (multiples of
# 64 share slots in a small set's table, so a merged set's order depends on how it was built and can differ from a flat
# replay's), into=dict `dict_value(h)`.  Rows are
# ``[key, window_id, tag, payload]``: ``E`` the container as a list (dict: its ``[k, v]`` items), ``L`` the value (dict:
# ``[k, v]``), ``M`` ``[open_us, close_us, sorted merged ids]``.

def set_value(h: int) -> int:
    return h * 64


def value_fn(into: str):
    return {"list": lambda h: h, "set": set_value, "dict": dict_value}[into]


def _json(v):
    return list(v) if isinstance(v, tuple) else v


def container_json(c):
    return [list(kv) for kv in c.items()] if isinstance(c, dict) else list(c)


def golden_rows(into: str, acts):
    """The restatement's rows (handles and intervals) as golden rows: each session's container built by ``container``."""
    vo = value_fn(into)
    out = []
    for rows in acts:
        act = []
        for k, w, tag, p in rows:
            if tag == "E":
                act.append([k, w, "E", container_json(container(into, p[0], p[1], vo))])
            elif tag == "L":
                act.append([k, w, "L", _json(vo(p))])
            else:
                act.append([k, w, "M", p])
        out.append(act)
    return out


def drive(builder, steps, now_box, us, dt, into: str):
    """Drive a `_WindowLogic` builder -- the reference's or this repository's -- through ``steps`` with the engine rules
    of src/operators.rs:755-806 (ascending key string per activation; a session logic is never discarded), :808-858
    (notify: every key whose ``notify_at()`` has come) and :862-894 (EOF).  ``now_box[0]`` is its clock's now.  Returns
    the golden rows per step, then EOF, and the number of merges (the merged ids of the meta rows)."""
    vo = value_fn(into)
    logics, acts = {}, []

    def conv(ks, res, rows):
        events, done = res
        assert not done  # session state is never discarded (windowing.py:798-806)
        for wid, tag, p in events:
            if tag == "E":
                rows.append([int(ks), wid, "E", container_json(p)])
            elif tag == "L":
                rows.append([int(ks), wid, "L", _json(p)])
            else:
                rows.append([int(ks), wid, "M", [us(p.open_time), us(p.close_time), sorted(p.merged_ids)]])

    for step in steps:
        now_box[0] = dt(step[1])
        rows = []
        if step[0] == "batch":
            grouped = {}
            for k, v in zip(step[2], step[4]):
                grouped.setdefault(key_str(k), []).append(vo(v))
            for ks in sorted(grouped):
                logic = logics.get(ks)
                if logic is None:
                    logic = logics[ks] = builder(None)
                conv(ks, logic.on_batch(grouped[ks]), rows)
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now_box[0]:
                    conv(ks, logics[ks].on_notify(), rows)
        acts.append(rows)
    rows = []
    for ks in sorted(logics):
        conv(ks, logics[ks].on_eof(), rows)
    acts.append(rows)
    return acts, sum(len(r[3][2]) for act in acts for r in act if r[2] == "M")


def builder_of(win, op, Dataflow, TestingSource, find, spec, steps, into: str, now_box, dt):
    """The `stateful_batch` builder of a `collect_window` flow over `SessionWindower` built with the operator modules
    given (the reference's, or this repository's): its EventClock reads each value's ts from the steps."""
    vo = value_fn(into)
    ts_of = {vo(v): t for s in steps if s[0] == "batch" for t, v in zip(s[3], s[4])}
    wait = timedelta.max if spec["wait_us"] == WAIT_FOREVER else timedelta(microseconds=spec["wait_us"])
    clock = win.EventClock(lambda v: dt(ts_of[v]), wait_for_system_duration=wait, now_getter=lambda: now_box[0])
    flow = Dataflow("g")
    up = op.key_on("k", op.input("in", flow, TestingSource([])), lambda _v: "k")
    win.collect_window("c", up, clock, win.SessionWindower(gap=timedelta(microseconds=spec["gap_us"])),
                       into={"list": list, "set": set, "dict": dict}[into], ordered=spec["ordered"])
    return find(flow).builder
