"""CPU restatement of `join_window` with insert modes first / last over session windows, on integer microseconds.
TEST INFRASTRUCTURE ONLY.

What the CUDA session join (``bw_sjwin``, csrc/bw_sjwin.cuh) replaces, restated in plain Python over value HANDLES
(paths relative to the bytewax v0.21.1 source tree):

* ``join_window``          -> pysrc/bytewax/operators/windowing.py:2056-2140 (sides labelled, clock sees the value)
* ``_JoinWindowLogic``     -> windowing.py:1849-1902 (``on_merge`` :1879-1891: "first" takes the merged-away session's
                              value where it is set, "last" keeps the survivor's), ``_JoinState`` operators/__init__.py
* ``_WindowLogic``         -> windowing.py:1046-1190 (late test, queue, ordered flush, inserts, merges, close, notify_at)
* ``SessionWindower``      -> windowing.py:671-810 (``tests.session_oracle.SessionWindower``); never discarded
* ``EventClock``           -> windowing.py:230-310 (``oracle.pyoracle.EventClock``)
* engine                   -> src/operators.rs:755-806 (ascending key string per activation), :808-858 (notify),
                              :862-894 (EOF)

``tools/gen_session_join_golden.py`` drives the reference's own classes and writes
``tests/golden/session_join_cases.json``; ``tests/test_oracle_session_join.py`` checks this restatement against it.
Rows are ``[key, window_id, tag, payload]`` in the order the reference's logic returns them: ``E`` carries the joined
tuple as a list (``None`` for an unset side), ``L`` ``[side, value]`` (window -1), ``M`` ``[open_us, close_us, sorted
merged ids]``.

Besides the rows, ``run_session_join`` reports the handles each call RELEASES, the contract of
``bw_sjwin_rows.released``: those no session and no queue entry of their key holds after the call, among the ones held
before it and the ones the call received.
"""

from __future__ import annotations

from typing import Dict, List, Optional, Tuple

from oracle.pyoracle import UTC_MAX_US, UTC_MIN_US, EventClock, key_str
from tests.session_oracle import LATE_SESSION_ID, SessionWindower

WAIT_FOREVER = (1 << 63) - 1  # BW_WAIT_FOREVER: the watermark never advances on data
S = 1_000_000
A = 1_640_995_200_000_000  # 2022-01-01T00:00:00Z
MODES = [(i, e) for i in ("first", "last") for e in ("complete", "final", "running")]


class SessionJoinLogic:
    """``_WindowLogic`` over a session windower and ``_JoinWindowLogic`` per session, for one key."""

    def __init__(self, spec: dict, now_us: int):
        self.insert_mode, self.emit_mode = spec["insert_mode"], spec["emit_mode"]
        self.ordered, self.sides = spec["ordered"], spec["sides"]
        self.clock = EventClock(spec["wait_us"], now_us)
        self.windower = SessionWindower(spec["gap_us"])
        self.states: Dict[int, List[Optional[int]]] = {}  # session id -> value per side (None: unset)
        self.queue: List[Tuple[Tuple[int, int], int]] = []  # ((side, value), ts)
        self.last_watermark = UTC_MIN_US
        self.merges = 0

    def _check_emit(self, st: List[Optional[int]]) -> List[list]:
        if self.emit_mode == "complete" and all(v is not None for v in st):
            row = list(st)
            for i in range(len(st)):
                st[i] = None  # _JoinState.clear
            return [row]
        if self.emit_mode == "running":
            return [list(st)]
        return []

    def _on_value(self, st: List[Optional[int]], side: int, value) -> List[list]:
        # windowing.py:1866-1876
        if self.insert_mode == "first" and st[side] is None:
            st[side] = value
        elif self.insert_mode == "last":
            st[side] = value
        return self._check_emit(st)

    def _on_merge(self, into: List[Optional[int]], orig: List[Optional[int]]) -> List[list]:
        # windowing.py:1879-1891
        for s in range(self.sides):
            if self.insert_mode == "first":
                if orig[s] is not None:  # self.state |= original.state
                    into[s] = orig[s]
            elif into[s] is None:  # original.state |= self.state; self.state = original.state
                into[s] = orig[s]
        return self._check_emit(into)

    def _flush(self, watermark: int) -> List[list]:
        # windowing.py:1095-1108
        if self.ordered:
            due = [e for e in self.queue if e[1] <= watermark]
            self.queue = [e for e in self.queue if not (e[1] <= watermark)]
            due.sort(key=lambda e: e[1])  # stable
        else:
            due, self.queue = self.queue, []
        events = []
        for (side, value), ts in due:  # _handle_inserts, windowing.py:1064-1077
            wid = self.windower.open_for(ts)
            st = self.states.setdefault(wid, [None] * self.sides)
            events.extend([wid, "E", row] for row in self._on_value(st, side, value))
        for orig, into in self.windower.merged():  # _handle_merged, windowing.py:1079-1085
            self.merges += 1
            events.extend([into, "E", row] for row in self._on_merge(self.states[into], self.states.pop(orig)))
        for wid, meta in self.windower.close_for(watermark):  # _handle_closed, windowing.py:1087-1093
            st = self.states.pop(wid)
            if self.emit_mode == "final":
                events.append([wid, "E", list(st)])
            events.append([wid, "M", [meta[0], meta[1], sorted(meta[2])]])
        return events

    def on_batch(self, items) -> List[list]:
        """``items``: ``(side, value, ts_us)`` in arrival order (windowing.py:1115-1133)."""
        self.clock.before_batch()
        events = []
        watermark = self.last_watermark
        for side, value, ts in items:
            _, watermark = self.clock.on_item(ts)
            self.last_watermark = watermark
            if ts < watermark:
                events.append([LATE_SESSION_ID, "L", [side, value]])
            else:
                self.queue.append(((side, value), ts))
        return events + self._flush(watermark)

    def on_notify(self) -> List[list]:
        watermark = self.clock.on_notify()  # windowing.py:1135-1142
        self.last_watermark = watermark
        return self._flush(watermark)

    def on_eof(self) -> List[list]:
        self.last_watermark = UTC_MAX_US  # windowing.py:1144-1151
        return self._flush(UTC_MAX_US)

    def notify_at(self) -> Optional[int]:
        # windowing.py:1153-1180 with an identity `to_system_utc`: the earliest close + gap, or the ts of queue[0]
        at = self.windower.notify_at()
        if self.ordered and self.queue:
            q = self.queue[0][1]
            at = q if at is None else min(at, q)
        return at

    def held(self) -> set:
        out = {v for st in self.states.values() for v in st if v is not None}
        out.update(e[0][1] for e in self.queue)
        return out


def run_session_join(spec: dict, steps, eof: bool = True, stats: Optional[dict] = None):
    """``spec``: insert_mode, emit_mode, ordered, sides, gap_us, wait_us.  ``steps``: ``["batch", now_us, keys, ts, sides,
    values]`` (one activation, ``now_getter() == now_us``) or ``["notify", now_us]`` (every key whose ``notify_at()`` has
    come, src/operators.rs:808-858).  Values must be distinct ints (the handles).  ``stats``: gets ``merges``.

    Returns ``(acts, released)``: the rows of every step (then EOF), and per step the sorted handles it released."""
    logics: Dict[str, SessionJoinLogic] = {}  # never discarded (windowing.py:798-806)
    ids: Dict[str, int] = {}
    acts, released = [], []
    held: set = set()

    def rows_of(ks, events):
        return [[ids[ks], wid, tag, payload] for wid, tag, payload in events]

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
            for k, t, sd, v in zip(step[2], step[3], step[4], step[5]):
                ks = key_str(k)
                ids[ks] = int(k)
                grouped.setdefault(ks, []).append((int(sd), v, int(t)))
                incoming.add(v)
            for ks in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
                lg = logics.get(ks)
                if lg is None:
                    lg = logics[ks] = SessionJoinLogic(spec, now)
                rows.extend(rows_of(ks, lg.on_batch(grouped[ks])))
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now:
                    rows.extend(rows_of(ks, logics[ks].on_notify()))
        settle(rows, incoming)
    if eof:
        rows = []
        for ks in sorted(logics):
            rows.extend(rows_of(ks, logics[ks].on_eof()))
        settle(rows, set())
    if stats is not None:
        stats["merges"] = sum(lg.merges for lg in logics.values())
    return acts, released


def seeded_spec(seed: int) -> dict:
    insert_mode, emit_mode = MODES[seed % 6]
    ordered = (seed // 6) % 2 == 0
    sides = 1 + (seed // 3) % 4
    gap = (0, S, 2 * S, 5 * S)[(seed // 2) % 4]
    wait = (0, S, 3 * S, WAIT_FOREVER)[(seed // 5) % 4]
    if gap == 0 and wait == WAIT_FOREVER:  # nothing would close before EOF: a key would need too many sessions
        wait = 3 * S
    return dict(insert_mode=insert_mode, emit_mode=emit_mode, ordered=ordered, sides=sides, gap_us=gap, wait_us=wait)


def seeded_steps(seed: int, n_steps: int = 30, n_keys: int = 6, moving: bool = True):
    """A seeded stream of activations and notify steps: keys 0..n_keys, timestamps jittered by +-4 s around a base that
    moves forward 1 s per activation, one item in ten up to 30 s behind.  Values are running integers (the handles).
    ``moving``: the system clock steps forward and some steps are notify phases; otherwise it is frozen."""
    import random

    rnd = random.Random(11000 + seed)
    spec = seeded_spec(seed)
    now, base, steps, nxt = A + 50 * S, A, [], 0
    for _ in range(n_steps):
        if moving:
            now += rnd.randint(0, 3 * S)
        if moving and rnd.random() < 0.25:
            steps.append(["notify", now])
            continue
        n = rnd.randint(1, 25)
        keys = [rnd.randint(0, n_keys) for _ in range(n)]
        ts = [base + rnd.randint(-4 * S, 4 * S) - (rnd.randint(5 * S, 30 * S) if rnd.random() < 0.1 else 0) for _ in range(n)]
        sides = [rnd.randrange(spec["sides"]) for _ in range(n)]
        steps.append(["batch", now, keys, ts, sides, list(range(nxt, nxt + n))])
        nxt += n
        base += S
    return spec, steps


SEEDED = range(48)
