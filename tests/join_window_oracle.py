"""CPU restatement of `join_window` with insert modes first / last on integer microseconds.  TEST INFRASTRUCTURE ONLY.

What the CUDA windowed join (``bw_jwin``, csrc/bw_jwin.cuh) replaces, restated in plain Python over value HANDLES
(paths relative to the bytewax v0.21.1 source tree):

* ``join_window``          -> pysrc/bytewax/operators/windowing.py:2056-2140 (sides labelled, clock sees the value)
* ``_JoinWindowLogic``     -> windowing.py:1849-1902, ``_JoinState`` operators/__init__.py:2076-2120
* ``_WindowLogic``         -> windowing.py:1046-1190 (late test, queue, ordered flush, inserts, close, notify_at)
* ``SlidingWindower``      -> windowing.py:603-668 (``oracle.pyoracle.SlidingWindower``; tumbling == offset == length)
* ``EventClock``           -> windowing.py:230-310 (``oracle.pyoracle.EventClock``)
* engine                   -> src/operators.rs:755-806 (ascending key string per activation, discard of empty logics),
                              :808-858 (notify), :862-894 (EOF)

``tools/gen_join_window_golden.py`` drives the reference's own classes and writes ``tests/golden/join_window_cases.json``;
``tests/test_oracle_join_window.py`` checks this restatement against it.  Rows are ``[key, window_id, tag, payload]`` in
the order the reference's logic returns them: ``E`` carries the joined tuple as a list (``None`` for an unset side),
``L`` ``[side, value]``, ``M`` ``[open_us, close_us]``.

Besides the rows, ``run_join_window`` reports the handles each call RELEASES: those that no window and no queue entry
of their key holds after the call, among the ones held before it and the ones the call received.  That is the contract
of ``bw_jwin_rows.released``; the reference keeps Python objects and has no such notion.
"""

from __future__ import annotations

from typing import Dict, List, Optional, Tuple

from oracle.pyoracle import UTC_MAX_US, EventClock, SlidingWindower, key_str

WAIT_FOREVER = (1 << 63) - 1  # BW_WAIT_FOREVER: the watermark never advances on data
S = 1_000_000
A = 1_640_995_200_000_000  # 2022-01-01T00:00:00Z
MODES = [(i, e) for i in ("first", "last") for e in ("complete", "final", "running")]


class JoinWindowLogic:
    """``_WindowLogic`` over a sliding windower and ``_JoinWindowLogic`` per window, for one key."""

    def __init__(self, spec: dict, now_us: int):
        self.insert_mode, self.emit_mode = spec["insert_mode"], spec["emit_mode"]
        self.ordered, self.sides = spec["ordered"], spec["sides"]
        self.clock = EventClock(spec["wait_us"], now_us)
        self.windower = SlidingWindower(spec["length_us"], spec["offset_us"], spec["align_us"])
        self.states: Dict[int, List[Optional[int]]] = {}  # window id -> value per side (None: unset)
        self.queue: List[Tuple[Tuple[int, int], int]] = []  # ((side, value), ts)
        self.last_watermark = -(1 << 62)

    def _on_value(self, st: List[Optional[int]], side: int, value) -> List[list]:
        # windowing.py:1866-1876
        if self.insert_mode == "first" and st[side] is None:
            st[side] = value
        elif self.insert_mode == "last":
            st[side] = value
        if self.emit_mode == "complete" and all(v is not None for v in st):
            row = list(st)
            for i in range(len(st)):
                st[i] = None
            return [row]
        if self.emit_mode == "running":
            return [list(st)]
        return []

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
            for wid in self.windower.open_for(ts):
                st = self.states.setdefault(wid, [None] * self.sides)
                events.extend([wid, "E", row] for row in self._on_value(st, side, value))
        for wid, meta in self.windower.close_for(watermark):  # _handle_closed, windowing.py:1087-1093
            st = self.states.pop(wid)
            if self.emit_mode == "final":
                events.append([wid, "E", list(st)])
            events.append([wid, "M", [meta[0], meta[1]]])
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
                events.extend([wid, "L", [side, value]] for wid in self.windower.late_for(ts))
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
        # windowing.py:1153-1180 with an identity `to_system_utc`: the earliest close, or the ts of queue[0] (ordered)
        at = min((m[1] for m in self.windower.opened.values()), default=None)
        if self.ordered and self.queue:
            q = self.queue[0][1]
            at = q if at is None else min(at, q)
        return at

    def is_empty(self) -> bool:
        # windowing.py:1110-1113
        return not self.states and not self.queue and self.windower.is_empty()

    def held(self) -> set:
        out = {v for st in self.states.values() for v in st if v is not None}
        out.update(e[0][1] for e in self.queue)
        return out


def run_join_window(spec: dict, steps, eof: bool = True):
    """``spec``: insert_mode, emit_mode, ordered, sides, length_us, offset_us, align_us, wait_us.  ``steps``:
    ``["batch", now_us, keys, ts, sides, values]`` (one activation, ``now_getter() == now_us``) or ``["notify", now_us]``
    (every key whose ``notify_at()`` has come, src/operators.rs:808-858).  Values must be distinct ints (the handles).

    Returns ``(acts, released)``: the rows of every step (then EOF), and per step the sorted handles it released."""
    logics: Dict[str, JoinWindowLogic] = {}
    ids: Dict[str, int] = {}
    acts, released = [], []
    held: set = set()

    def rows_of(ks, events):
        return [[ids[ks], wid, tag, payload] for wid, tag, payload in events]

    def finish(ks, lg, rows, events):
        rows.extend(rows_of(ks, events))
        if lg.is_empty():
            del logics[ks]  # src/operators.rs:796-799: the clock state goes too

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
                    lg = logics[ks] = JoinWindowLogic(spec, now)
                finish(ks, lg, rows, lg.on_batch(grouped[ks]))
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now:
                    lg = logics[ks]
                    finish(ks, lg, rows, lg.on_notify())
        settle(rows, incoming)
    if eof:
        rows = []
        for ks in sorted(logics):
            lg = logics[ks]
            finish(ks, lg, rows, lg.on_eof())
        settle(rows, set())
    return acts, released


def seeded_spec(seed: int) -> dict:
    insert_mode, emit_mode = MODES[seed % 6]
    ordered = (seed // 6) % 2 == 0
    sides = 1 + (seed // 3) % 4
    length, offset = ((4 * S, 4 * S), (6 * S, 2 * S), (5 * S, 3 * S), (3 * S, 3 * S))[(seed // 2) % 4]
    wait = (0, S, 3 * S, WAIT_FOREVER)[(seed // 5) % 4]
    align = A + (seed % 7) * 333_333
    return dict(insert_mode=insert_mode, emit_mode=emit_mode, ordered=ordered, sides=sides, length_us=length, offset_us=offset,
                align_us=align, wait_us=wait)


def seeded_steps(seed: int, n_steps: int = 30, n_keys: int = 6, moving: bool = True):
    """A seeded stream of activations and notify steps: keys 0..n_keys, timestamps jittered by +-4 s around a base that
    moves forward 1 s per activation, one item in ten up to 30 s behind.  Values are running integers (the handles).
    ``moving``: the system clock steps forward and some steps are notify phases; otherwise it is frozen."""
    import random

    rnd = random.Random(7000 + seed)
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
