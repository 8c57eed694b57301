"""Streams for the window fold under a moving system clock, with the shapes they claim to reach.  CPU only.

A case is a list of steps:
  ("batch", now, keys, ts, ids)    `now_getter()` is `now`, one activation, then its rows
  ("ingest", now, keys, ts, ids)   the same activation; its rows come out with the next step's (no advance between)
  ("set_now", now)                 the clock moves with no activation and no notify phase
  ("notify", now)                  the notify phase at system time `now` (src/operators.rs:808-858)
and EOF after the last step.  `ids` number the rows of a case from 0; a test maps them to values of its type.

`run` drives oracle/pyoracle.StatefulBatchEngine (its clock is pinned to the reference by
tests/golden/system_time_cases.json) through the steps and records per step the rows and the SHAPES the step met:
the key-state, due-boundary, drift and limit cases of the notify phase (`k_close_wake`) and of a moving-clock
activation.  Every builder names the shapes it must reach and tests/test_oracle_clock.py checks them, so a builder
that stops reaching a shape fails on the CPU instead of passing quietly on the GPU.

The device never lets its system time go backwards (windowing.py:250-261) and runs a notify phase at the largest
system time it has seen; `run` drives the oracle's notify phase at that same time."""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Set

import numpy as np

from oracle import pyoracle as po

S = 1_000_000
A = 1_640_995_200_000_000          # align_to: 2022-01-01T00:00:00Z
NOW26 = 1_780_000_000_000_000      # a wall clock in 2026 (2026-05-28T20:26:40Z)
UTC_MIN, UTC_MAX = po.UTC_MIN_US, po.UTC_MAX_US
FOREVER = (1 << 63) - 1            # BW_WAIT_FOREVER
KMAX = 2**64 - 1                   # BW_EMPTY_KEY: its table slot is the alias slot at index capacity
K20 = 10**19 + 7                   # a 20-digit key


@dataclass
class Case:
    name: str
    steps: list
    claims: Dict[int, Set[str]]       # step index -> shapes the step must meet
    red: str = "sum"
    length: int = 10 * S
    offset: Optional[int] = None
    wait: int = 0
    ordered: bool = False
    align: int = A
    refuse_at: Optional[int] = None   # an ordered fold's device refuses this notify phase (BW_ERR_STATE)

    def spec(self, red: Optional[str] = None, ordered: Optional[bool] = None) -> po.FoldSpec:
        return po.FoldSpec(red or self.red, self.length, self.offset, self.align, self.wait,
                           self.ordered if ordered is None else ordered)

    @property
    def n_rows(self) -> int:
        return sum(len(s[2]) for s in self.steps if s[0] in ("batch", "ingest"))


@dataclass
class Trace:
    rows: List[list] = field(default_factory=list)     # per step, then EOF: (key, wid, tag, payload)
    shapes: List[Set[str]] = field(default_factory=list)
    refuse: List[bool] = field(default_factory=list)   # per step: k_close_wake's ordered refusal rule holds
    live_after: List[Set[int]] = field(default_factory=list)
    due_frac: List[float] = field(default_factory=list)


# ---------------------------------------------------------------------------------------------- oracle state, read


def windows_of(logic) -> Dict[int, int]:
    """wid -> close of every window the key holds: the opened ones and those of its queued items (the device folds
    an ordered key's items at once; only the reference queues them)."""
    out = {w: m[1] for w, m in logic.windower.opened.items()}
    for _v, t in logic.queue:
        for w in logic.windower.intersects(t):
            out.setdefault(w, logic.windower.metadata_for(w)[1])
    return out


def watermark_at(logic, now: int) -> int:
    c = logic.clock
    return c.watermark_base + (max(now, c._system_now) - c.system_time_of_max_event)


def led_by(logic, wait: int) -> Optional[int]:
    """max_j(ts_j - now_j) over the key's items (the device's max_ts in the frame of now), once an item set the
    watermark (before that the base is UTC_MIN)."""
    c = logic.clock
    if c.watermark_base == UTC_MIN:
        return None
    return c.watermark_base + wait - c.system_time_of_max_event


def refuses(case: Case, eng, now: int) -> bool:
    """k_close_wake's refusal on an ordered fold: some key's items led the system clock (max_ts > 0 in the frame of
    now) and this notify's drifted watermark closes one of its windows.  Only there can the reference's extra wake-up
    at its queue head (windowing.py:1154-1180) change what a notify phase emits."""
    if not case.ordered or not (0 < case.wait < FOREVER):
        return False
    for logic in eng.logics.values():
        led, ws = led_by(logic, case.wait), windows_of(logic)
        if led is not None and led > 0 and ws and min(ws.values()) <= watermark_at(logic, now):
            return True
    return False


def _notify_shapes(case: Case, pre, now: int, rows, emitted_before: Dict[int, Set[int]]):
    """`pre`: per live key before the notify phase (key, windows, watermark at now, max_ts, queued?, scheduled at)."""
    sh: Set[str] = set()
    tumbling = case.offset is None or case.offset == case.length
    emitted: Dict[int, Set[int]] = {}
    for k, w, tag, _p in rows:
        if tag == "E":
            emitted.setdefault(k, set()).add(w)
    n_live = n_due = 0
    for k, ws, wm, led, queued, sched in pre:
        if not ws:
            continue
        n_live += 1
        first = min(ws.values())
        due = first <= now  # k_close_wake's due test
        n_due += due
        if not case.ordered or not queued:
            assert due == (sched is not None and sched <= now), (k, first, sched, now)  # == the reference's schedule
        ids = sorted(ws)
        if tumbling:
            shape = {1: "pane0_only", 2: "p1_prev" if ids[-1] == ids[0] + 1 else "two_apart"}.get(len(ids), "list")
            sh.add(shape)
        elif emitted_before.get(k):
            sh.add(f"sliding_partial_{case.length // S}_{case.offset // S}")
        if first == now:
            sh.add("close_eq_now")
        if first == now + 1:
            sh.add("close_now_plus_1")
        em = emitted.get(k, set())
        if due and not em and wm < first:
            sh.add("due_wm_held")
        if due and em and len(em) < len(ids):
            sh.add("due_partial")
        if due and em and len(em) == len(ids):
            sh.add("due_all")
        if k == KMAX:
            sh.add("alias_key_due" if due else "alias_key")
        if k >= 10**19:
            sh.add("key20_due" if due else "key20")
        if first - case.length < UTC_MIN + now - A:
            sh.add("near_utc_min")
        if max(ws.values()) > UTC_MAX - 3600 * S:
            sh.add("near_utc_max")
        if led is not None and led > 0:
            sh.add("event_time_leads")
    if n_live and not emitted:
        sh.add("notify_noop")
    if n_live == 0:
        sh.add("notify_empty")
    return sh, (n_due / n_live if n_live else 0.0)


def _batch_shapes(case: Case, keys, ts, rows, pre, gone, now) -> Set[str]:
    """`pre`: key string -> (watermark at now, frozen watermark (no drift), windows) before the activation."""
    sh: Set[str] = set()
    per: Dict[int, list] = {}
    for k, t in zip(keys, ts):
        per.setdefault(k, []).append(t)
    tags: Dict[int, list] = {}
    for k, _w, tag, _p in rows:
        tags.setdefault(k, []).append(tag)
    for k, tl in per.items():
        ks, tg = po.key_str(k), tags.get(k, [])
        if ks in pre:
            wm, frozen, ws = pre[ks]
            if len(tl) == 1 and tg[:1] == ["L"] and "E" in tg and tl[0] >= frozen:
                sh.add("drift_late_closes")  # late only because the watermark drifted, and it closes
            if ws and "E" in tg and "L" not in tg and max(frozen, max(tl) - case.wait) < min(ws.values()):
                sh.add("drift_touch_closes")  # its own rows prove nothing closable; the drift does
        elif k in gone and "L" not in tg:
            sh.add("comeback")
        if k == KMAX:
            sh.add("alias_key_batch")
    if case.wait == 0 and all(t == now for t in ts):
        sh.add("system_clock_shaped")
    if any(UTC_MIN <= t < UTC_MIN + case.wait + now for t in ts) and not any(tag == "L" for tg in tags.values() for tag in tg):
        sh.add("below_frame_floor_on_time")  # late under a floor of UTC_MIN in the frame of now
    return sh


def run(case: Case, vals_of: Optional[Callable] = None, red: Optional[str] = None,
        ordered: Optional[bool] = None) -> Trace:
    """Drive the oracle through the case.  `vals_of(ids)` gives the values it folds (default: the ids)."""
    eng = po.StatefulBatchEngine(case.spec(red, ordered))
    c = case if ordered is None else Case(**{**case.__dict__, "ordered": ordered})
    tr = Trace()
    kept = None  # the device's system time: it never goes backwards
    emitted_before: Dict[int, Set[int]] = {}
    carried: list = []
    for st in case.steps:
        kind, sh, ref, frac = st[0], set(), False, 0.0
        if kind in ("batch", "ingest"):
            _, now, keys, ts, ids = st
            kept = now if kept is None else max(kept, now)
            eng.set_now(kept)
            keys, ts = [int(k) for k in keys], [int(t) for t in ts]
            pre = {ks: (watermark_at(lg, kept), lg.clock.watermark_base, windows_of(lg)) for ks, lg in eng.logics.items()}
            gone = {eng._keys[ks] for ks in eng._keys if ks not in eng.logics}
            vals = vals_of(ids) if vals_of else [int(i) for i in ids]
            rows = eng.on_batch(keys, ts, vals)
            sh = _batch_shapes(c, keys, ts, rows, pre, gone, kept)
            rows = carried + rows
            carried, rows = (rows, []) if kind == "ingest" else ([], rows)
        elif kind == "set_now":
            kept = st[1] if kept is None else max(kept, st[1])
            eng.set_now(kept)
            sh.add("set_now")
            rows = []
        else:
            if kept is None:
                sh.add("notify_before_ingest")
            elif st[1] < kept:
                sh.add("clock_backwards")
            elif st[1] == kept:
                sh.add("clock_still")
            if carried:
                sh.add("notify_after_ingest")
            kept = st[1] if kept is None else max(kept, st[1])
            ref = refuses(c, eng, kept)
            pre = [(eng._keys[ks], windows_of(lg), watermark_at(lg, kept), led_by(lg, case.wait), bool(lg.queue),
                    eng.sched.get(ks)) for ks, lg in eng.logics.items()]
            rows = carried + eng.on_notify(kept)
            carried = []
            ns, frac = _notify_shapes(c, pre, kept, rows, emitted_before)
            sh |= ns
        for k, w, tag, _p in rows:
            if tag == "E":
                emitted_before.setdefault(k, set()).add(w)
        tr.rows.append(rows)
        tr.shapes.append(sh)
        tr.refuse.append(ref)
        tr.due_frac.append(frac)
        tr.live_after.append({eng._keys[ks] for ks in eng.logics})
    tr.rows.append(carried + eng.on_eof())
    return tr


# ---------------------------------------------------------------------------------------------- builders


class _B:
    """Accumulates steps; row ids number the rows of the case."""

    def __init__(self):
        self.steps, self.claims, self.nid = [], {}, 0

    def _rows(self, kind, now, kt, claim):
        keys = np.array([k for k, _ in kt], np.uint64)
        ts = np.array([t for _, t in kt], np.int64)
        ids = np.arange(self.nid, self.nid + len(kt), dtype=np.int64)
        self.nid += len(kt)
        self.steps.append((kind, int(now), keys, ts, ids))
        self._claim(claim)

    def batch(self, now, kt, *claim):
        self._rows("batch", now, kt, claim)

    def ingest(self, now, kt, *claim):
        self._rows("ingest", now, kt, claim)

    def notify(self, now, *claim):
        self.steps.append(("notify", int(now)))
        self._claim(claim)

    def set_now(self, now, *claim):
        self.steps.append(("set_now", int(now)))
        self._claim(claim)

    def _claim(self, claim):
        if claim:
            self.claims[len(self.steps) - 1] = set(claim)

    @property
    def last(self):
        return len(self.steps) - 1


def key_states() -> Case:
    """Tumbling 10 s windows, wait 45 s, event time a little behind the clock.  At the notify phases: keys holding one
    pane, two adjacent panes (pane 1 as the previous pane), two panes apart and three or more (an overflow list); the
    alias-slot key and a 20-digit key; a key due exactly at its close (close == now) and one a microsecond short of
    it; due keys the wait still holds, due keys closing some and all of their windows; a discarded key that comes
    back older; a notify with the clock standing still and one with the clock behind."""
    b, T = _B(), A + 1000 * S  # T: a window boundary
    b.notify(T - 60 * S, "notify_before_ingest", "notify_empty")
    b.batch(T, [(1, T - 5 * S), (2, T - 15 * S), (2, T - 5 * S), (3, T - 35 * S), (3, T - 25 * S), (3, T - 15 * S),
                (3, T - 1 * S), (4, T - 25 * S), (4, T - 5 * S), (KMAX, T - 5 * S), (K20, T - 5 * S), (6, T - 36 * S)])
    b.notify(T, "clock_still", "close_eq_now", "due_wm_held", "pane0_only", "p1_prev", "two_apart", "list",
             "alias_key_due", "key20_due", "notify_noop")
    b.batch(T + 1 * S, [(5, T + 1 * S), (7, T - 9 * S), (7, T + 1 * S)])  # (5: its one window closes at T + 10 s)
    b.notify(T + 10 * S - 1, "close_now_plus_1")
    b.notify(T + 20 * S, "due_partial")
    b.notify(T + 5 * S, "clock_backwards")
    b.notify(T + 50 * S, "due_all")
    b.batch(T + 51 * S, [(1, T - 3 * S), (6, T - 50 * S)], "comeback")
    b.notify(T + 70 * S)
    return Case("key_states", b.steps, b.claims, wait=45 * S)


def sliding_partial(length: int, offset: int) -> Case:
    """Sliding windows: keys whose windows close over several notify phases, so `closed_upto` is partly emitted when
    k_close_wake tests them (the due test corrects the oldest pane's first window by it)."""
    b, T = _B(), A + 2000 * S
    kt = [(k, T - 40 * S + k * 3 * S + j * 7 * S) for k in range(1, 9) for j in range(5)]
    b.batch(T, kt)
    tag = f"sliding_partial_{length // S}_{offset // S}"
    for i, d in enumerate((5, 9, 14, 20, 27)):
        b.notify(T + d * S, *((tag,) if i >= 1 else ()))
    b.batch(T + 28 * S, [(3, T + 2 * S), (9, T + 20 * S)])
    b.notify(T + 40 * S)
    return Case(f"sliding_partial_{length // S}_{offset // S}", b.steps, b.claims, length=length, offset=offset,
                wait=20 * S)


def drift() -> Case:
    """Wait 2 s.  Key Z: an on-time row, then 14 s of system time later a single row 1 s newer -- late only because
    its watermark drifted; its window closes in that activation.  Key D: a row whose window's close the drift reaches
    exactly when D's next row arrives, a row that is not late and proves nothing closable by its own timestamp -- K4
    must still see D (a moving clock marks every touched key).  Then an ingest at one time, the clock moved with no
    advance, an ingest at the new time and the advance: the first activation folds in its own time's frame."""
    b, T = _B(), A + 3000 * S
    fill = [(100 + i, T - S + i * 10_000) for i in range(50)]
    b.batch(T, fill + [(11, T - 1 * S), (12, T - 8 * S)])
    b.batch(T + 10 * S, [(12, T + 1 * S)], "drift_touch_closes")
    b.batch(T + 14 * S, [(11, T)], "drift_late_closes")
    b.notify(T + 15 * S)
    b.ingest(T + 20 * S, [(13, T + 19 * S), (14, T + 18 * S)])
    b.set_now(T + 40 * S, "set_now")
    b.ingest(T + 40 * S, [(13, T + 25 * S), (14, T + 39 * S)])
    b.batch(T + 41 * S, [(15, T + 40 * S)])
    b.notify(T + 60 * S)
    return Case("drift", b.steps, b.claims, wait=2 * S)


def due_boundary() -> Case:
    """Wait 0, event time 4 s ahead of the clock: a key whose earliest close is 1 us after the notify phase is not
    woken although its drifted watermark has passed the close; at the next notify phase the close equals now, the key
    is woken and its window closes."""
    b, T = _B(), A + 3500 * S
    b.batch(T - 5 * S, [(1, T - 1 * S), (2, T - 2 * S)])
    b.notify(T - 1, "close_now_plus_1", "event_time_leads", "notify_noop")
    b.notify(T, "close_eq_now", "due_all")
    return Case("due_boundary", b.steps, b.claims, wait=0)


def sliding_lead() -> Case:
    """Sliding 10 / 5 s, wait 2 s, event time up to 14 s ahead of the clock: the first activation emits the key's first
    two windows, so `closed_upto` decides its next close (+15 s); at the notify phase at +10 s that close is not due
    (the first window over its oldest pane, already emitted, would be), although the drifted watermark passes it."""
    b, T = _B(), A + 3600 * S
    b.batch(T, [(1, T + 1 * S), (1, T + 6 * S), (1, T + 14 * S)])
    b.notify(T + 10 * S, "sliding_partial_10_5", "event_time_leads", "notify_noop")
    b.notify(T + 15 * S, "close_eq_now", "due_all")
    return Case("sliding_lead", b.steps, b.claims, offset=5 * S, wait=2 * S)


def drift_touch(offset: int) -> Case:
    """Wait 20 s.  A key holding two panes gets, once the drift has brought its watermark to the close of the older
    one, a row that is on time, lands in its newest pane (no pane is created) and proves nothing closable by its own
    timestamp, in a clean activation: only the drift closes the older window, so every path (the segment fold, also
    its general path for sliding windows, and the direct kernel) must hand the key to K4."""
    b, T = _B(), A + 3700 * S
    older = T - 12 * S if offset == 10 * S else T - 8 * S
    b.batch(T, [(1, older), (1, T - 3 * S), (2, T - 9 * S)])
    b.batch(T + 23 * S - offset, [(1, T - 5 * S if offset == 10 * S else T - 2 * S)], "drift_touch_closes")
    b.notify(T + 40 * S)
    return Case(f"drift_touch_10_{offset // S}", b.steps, b.claims, offset=offset, wait=20 * S)


def system_clock(n_steps: int = 12) -> Case:
    """A SystemClock-shaped stream: every row's timestamp is its batch's system time, wait 0; notify phases between."""
    b, T = _B(), A + 4000 * S + 300_000
    rnd = np.random.default_rng(41)
    for i in range(n_steps):
        now = T + i * 1_700_000
        b.batch(now, [(int(k), now) for k in rnd.integers(0, 40, 30)], "system_clock_shaped")
        if i % 3 == 2:
            b.notify(now + 900_000)
    return Case("system_clock", b.steps, b.claims, red="count", length=2 * S)


def wait_forever() -> Case:
    """wait = forever: no watermark moves; every notify phase is a no-op and everything closes at EOF."""
    b, T = _B(), A + 5000 * S
    b.batch(T, [(k, T - k * S) for k in range(1, 20)])
    b.notify(T + 100 * S, "notify_noop")
    b.batch(T + 200 * S, [(k, T + 150 * S) for k in range(1, 20, 2)])
    b.notify(T + 10_000 * S, "notify_noop")
    return Case("wait_forever", b.steps, b.claims, wait=FOREVER)


def wall_clock_2026(ordered: bool = False) -> Case:
    """A 2026 wall clock over 2022 event times, wait 3 s: every key is due at every notify phase and closes what its
    drifted watermark allows; event times that lead the clock are in `event_time_leads`."""
    b, T = _B(), NOW26
    rnd = np.random.default_rng(42)
    t0 = A + 7 * 86400 * S
    for i in range(6):
        now = T + i * 2 * S
        kt = [(int(k), t0 + i * 4 * S + int(d)) for k, d in zip(rnd.integers(0, 300, 400), rnd.integers(0, 4 * S, 400))]
        b.batch(now, kt)
        b.notify(now + S)
    return Case("wall_clock_2026" + ("_ordered" if ordered else ""), b.steps, b.claims, wait=3 * S, ordered=ordered)


def event_time_leads(ordered: bool) -> Case:
    """Event time 30 s ahead of the clock, wait 10 s.  Unordered: the notify phases agree with the reference.
    Ordered: the reference also wakes a key at its queue head; the device refuses the notify phase where that can
    change a row (`refuses`)."""
    b, T = _B(), A + 6000 * S
    b.batch(T, [(k, T + 30 * S + k * 100_000) for k in range(1, 30)])
    b.notify(T + 15 * S, "event_time_leads")
    b.notify(T + 25 * S, "event_time_leads")
    c = Case("event_time_leads" + ("_ordered" if ordered else ""), b.steps, b.claims, wait=10 * S, ordered=ordered)
    if ordered:
        c.refuse_at = 2
    return c


def ordered_queue_head(which: str) -> Case:
    """The ordered fold's queue-head wake-up.  `late_wake`: event time runs ahead of the clock by more than the wait;
    the reference emits windows 9 and 10 at the notify at +95 s, the windows' closes are later (the device would wait
    for EOF).  `early_wake`: the queue head leads the clock, a later arrival sits in a window whose close the drifted
    watermark reaches first; the reference waits for the head (+50 s), the close is due at +6 s.  `behind`: the same
    streams with event time behind the clock: the device and the reference agree, nothing is refused."""
    b = _B()
    if which == "late_wake":
        b.batch(A, [(1, A + 95 * S), (1, A + 100 * S)])
        b.notify(A + 95 * S)
        return Case("ordered_late_wake", b.steps, b.claims, wait=10 * S, ordered=True, refuse_at=1)
    T = A + 1000 * S
    if which == "early_wake":
        b.batch(T, [(1, T + 50 * S), (1, T - 45 * S)])
        b.notify(T + 6 * S)
        return Case("ordered_early_wake", b.steps, b.claims, length=S, wait=100 * S, ordered=True, refuse_at=1)
    b.batch(T, [(1, T - 50 * S), (1, T - 95 * S), (2, T - 3 * S), (2, T - 9 * S)])
    b.notify(T + 6 * S)
    b.notify(T + 60 * S)
    b.batch(T + 61 * S, [(2, T + 61 * S), (3, T + 20 * S)])
    b.notify(T + 95 * S)
    return Case("ordered_behind", b.steps, b.claims, length=S, wait=100 * S, ordered=True)


def limits() -> Case:
    """Timestamps at the ends of the range under a 2026 clock, wait 2 s: rows within `now + wait` of UTC_MIN (a
    floor of UTC_MIN in the frame of now made them late; the reference's floor is UTC_MIN itself), and rows near
    UTC_MAX that close only at EOF.  (The last window, [UTC_MAX + 1 - 10 s, UTC_MAX + 1), closes after UTC_MAX and so
    never in the reference; the rows near UTC_MAX stay in the windows before it.)"""
    b, T = _B(), NOW26
    lo = [(1, UTC_MIN + 86400 * S), (2, UTC_MIN + 1), (3, UTC_MIN + T - S), (1, UTC_MIN + 86400 * S + 5)]
    b.batch(T, lo, "below_frame_floor_on_time")
    b.batch(T + S, [(2, UTC_MIN + 3 * S), (4, UTC_MIN + 2 * S + 5)], "below_frame_floor_on_time")
    b.notify(T + 2 * S, "near_utc_min")
    b.batch(T + 3 * S, [(5, UTC_MAX - 15 * S), (6, UTC_MAX - 10 * S), (5, UTC_MAX - 30 * S)])
    b.notify(T + 4 * S, "near_utc_max")
    return Case("limits", b.steps, b.claims, wait=2 * S, align=0)


def emit_capacity() -> Case:
    """Wait 20 s: the notify phase at +25 s closes exactly 128 windows, and nothing emits a row before it."""
    b, T = _B(), A + 8000 * S
    b.batch(T, [(k, T - 5 * S) for k in range(1, 101)] + [(k, T - 15 * S) for k in range(1, 29)])
    b.notify(T + 25 * S)
    return Case("emit_capacity", b.steps, b.claims, wait=20 * S)


def many_keys(n_keys: int, frac: float, seed: int = 0) -> Case:
    """`n_keys` keys (random u64s), each with one row; a random `frac` of them in a window that closes by the notify
    phase, the rest in one that closes 1 us after it."""
    rnd = np.random.default_rng(seed)
    T = A + 9000 * S
    keys = np.unique(rnd.integers(0, 2**64 - 1, n_keys, dtype=np.uint64, endpoint=True))
    rnd.shuffle(keys)
    due = rnd.random(len(keys)) < frac
    ts = np.where(due, T - 5 * S, T + 5 * S).astype(np.int64)
    b = _B()
    b.steps.append(("batch", T, keys, ts, np.arange(len(keys), dtype=np.int64)))
    b.nid = len(keys)
    b.notify(T + 10 * S - 1)
    return Case(f"many_keys_{n_keys}_{frac}", b.steps, b.claims, red="count", wait=0)


def all_cases() -> List[Case]:
    return [key_states(), sliding_partial(10 * S, 5 * S), sliding_partial(10 * S, 4 * S), sliding_partial(9 * S, 3 * S),
            drift(), due_boundary(), sliding_lead(), drift_touch(10 * S), drift_touch(5 * S), system_clock(), wait_forever(), wall_clock_2026(False), wall_clock_2026(True),
            event_time_leads(False), event_time_leads(True), ordered_queue_head("late_wake"),
            ordered_queue_head("early_wake"), ordered_queue_head("behind"), limits(), emit_capacity()]


# ---------------------------------------------------------------------------------------------- the device's paths


def clean(rel_ts, gprev: int, wait: int) -> bool:
    """The streaming verdict: no row behind (the running maximum over everything ingested before it) - wait, in the
    frame of each activation's system time (ts - now); gprev, the maximum of the earlier activations' (ts - now)."""
    if wait >= FOREVER:
        return True
    m = gprev
    for t in rel_ts:
        if m != -(2**63) and t < m - wait:
            return False
        m = max(m, t)
    return True


def suspects(rel_ts, gprev: int, wait: int) -> int:
    """Rows behind (the running maximum before them) - wait: what the late split puts in its table."""
    n, m = 0, gprev
    for t in rel_ts:
        if m != -(2**63) and t < m - wait:
            n += 1
        m = max(m, t)
    return n


def activation_paths(case: Case) -> List[Optional[str]]:
    """Per step: None (not an activation); "none" (wait forever: no watermark, the direct kernel); "seg" (clean: the
    segment fold); "split" (late rows split off, at most max(1024, rows / 16) suspects); "sort" (more suspects, or
    rows spanning more than the segment fold's 32-bit relative timestamps)."""
    out, g, kept = [], -(2**63), None
    rows = max([len(s[2]) for s in case.steps if s[0] in ("batch", "ingest")] + [1])
    for st in case.steps:
        if st[0] in ("batch", "ingest"):
            kept = st[1] if kept is None else max(kept, st[1])
            rel = [int(t) - kept for t in st[3]]
            if case.wait >= FOREVER:
                out.append("none")
            elif clean(rel, g, case.wait):
                out.append("seg")
            else:
                few = suspects(rel, g, case.wait) <= max(1024, rows // 16)
                out.append("split" if few and max(rel) - min(rel) <= 0x7FFFFFF0 else "sort")
            g = max([g] + rel)
        else:
            if st[0] == "set_now":
                kept = st[1] if kept is None else max(kept, st[1])
            out.append(None)
    return out


# ---------------------------------------------------------------------------------------------- C1 size


def c1_stepping(n_rows: int, n_keys: int, n_acts: int, seed: int = 0, straggle: float = 0.01) -> Case:
    """C1-like activations under a wall-clock-like stepping clock, with a notify phase between every two: count over
    1 s tumbling windows, wait 0; activation b arrives at now_b = T + 0.7 s b and its rows carry now_b (the shape of a
    SystemClock source), except a random `straggle` of them sent 0.5 .. 2 s back (late when their key was seen before).
    Row values are their ids."""
    rnd = np.random.default_rng(seed)
    T = A + 10_000 * S + 123_457
    b, nid = _B(), 0
    for i in range(n_acts):
        now = T + i * 700_000
        keys = rnd.integers(0, n_keys, n_rows).astype(np.uint64)
        ts = np.full(n_rows, now, np.int64)
        back = rnd.random(n_rows) < straggle
        ts[back] -= rnd.integers(500_000, 2_000_000, int(back.sum()))
        b.steps.append(("batch", now, keys, ts, np.arange(nid, nid + n_rows, dtype=np.int64)))
        nid += n_rows
        b.notify(now + 350_000)
    return Case(f"c1_stepping_{n_rows}_{n_keys}", b.steps, b.claims, red="count", length=S, wait=0)


def _key_string_order(keys: np.ndarray, wids: np.ndarray, seq: np.ndarray) -> np.ndarray:
    """Ascending key string (src/operators.rs:758-767), then `seq` (window id, or arrival index)."""
    return np.lexsort((seq, wids, keys.astype(str)))


def c1_reference(case: Case):
    """The reference's rows for `c1_stepping` streams, vectorised: count, tumbling, wait 0, unordered, event time never
    ahead of the clock.  Per key the watermark is M + now with M = max(ts - now) over its items (windowing.py:263-302),
    reset when every window of the key has closed (the logic is discarded); an item is late iff ts - now < M before it;
    a batch closes its keys' windows up to M + now, a notify phase every key's (with wait 0 and M <= 0 a key with a
    closable window is always due).  Returns per step (and EOF): (down, late) with down = [(key, wid, count)] and late
    = [(key, wid, id, ts)], in the reference's order.  tests/test_oracle_clock.py checks it against the oracle."""
    NEG = -(2**62)
    n_keys = int(max(int(s[2].max()) for s in case.steps if s[0] == "batch")) + 1
    M = np.full(n_keys, NEG, np.int64)
    L, al = case.length, case.align
    open_k = np.zeros(0, np.int64)
    open_w = np.zeros(0, np.int64)
    open_c = np.zeros(0, np.int64)
    out = []

    def close(sel_keys_mask, wm_of_key):
        nonlocal open_k, open_w, open_c
        shut = sel_keys_mask[open_k] & (al + (open_w + 1) * L <= wm_of_key[open_k])
        k, w, c = open_k[shut], open_w[shut], open_c[shut]
        o = _key_string_order(k, w, w)
        open_k, open_w, open_c = open_k[~shut], open_w[~shut], open_c[~shut]
        live = np.zeros(n_keys, bool)
        live[open_k] = True
        M[sel_keys_mask & ~live] = NEG  # discarded with its watermark
        return [(int(a), int(b), int(x)) for a, b, x in zip(k[o], w[o], c[o])]

    for st in case.steps:
        if st[0] == "batch":
            _, now, keys, ts, ids = st
            k = keys.astype(np.int64)
            rel = ts - now
            o = np.argsort(k, kind="stable")
            ks, rs = k[o], rel[o]
            start = np.ones(len(ks), bool)
            start[1:] = ks[1:] != ks[:-1]
            seg = np.cumsum(start) - 1
            code = seg * (1 << 42) + (rs + (1 << 41))
            run = np.maximum.accumulate(code)
            excl = np.empty_like(run)
            excl[0] = -1
            excl[1:] = run[:-1]
            excl_rel = np.where(start, NEG, excl - seg * (1 << 42) - (1 << 41))
            before = np.maximum(M[ks], excl_rel)
            late_s = (before != NEG) & (rs < before)
            np.maximum.at(M, ks, rs)
            late = np.zeros(len(k), bool)
            late[o] = late_s
            wid = (ts - al) // L
            li = np.flatnonzero(late)
            lo = _key_string_order(k[li], np.zeros(len(li), np.int64), li)
            late_rows = [(int(k[i]), int(wid[i]), int(ids[i]), int(ts[i])) for i in li[lo]]
            ok = ~late
            code2 = np.concatenate([open_k * (1 << 40) + open_w, k[ok] * (1 << 40) + wid[ok]])
            cnt2 = np.concatenate([open_c, np.ones(int(ok.sum()), np.int64)])
            u, inv = np.unique(code2, return_inverse=True)
            open_c = np.bincount(inv, weights=cnt2).astype(np.int64)
            open_k, open_w = u >> 40, u & ((1 << 40) - 1)
            touched = np.zeros(n_keys, bool)
            touched[k] = True
            out.append((close(touched, M + now), late_rows))
        else:
            everyone = np.ones(n_keys, bool)
            out.append((close(everyone, M + st[1]), []))
    everyone = np.ones(n_keys, bool)
    out.append((close(everyone, np.full(n_keys, 2**62, np.int64)), []))
    return out


def many_keys_reference(case: Case):
    """The reference's rows for `many_keys` streams, vectorised (one row per key, count, wait 0): nothing closes in
    the activation (every row's window closes after it); the notify phase closes the windows that have closed by
    then (their keys are due: close <= now, and the watermark ts - now + now' reaches them), the rest close at EOF.
    Per step: (down, late) as `c1_reference` gives them."""
    (_, now, keys, ts, _ids), (_, t_notify) = case.steps
    wid = (ts - case.align) // case.length
    close = case.align + (wid + 1) * case.length
    shut = (close <= t_notify) & (close <= ts - now + t_notify)  # due, and reached by the drifted watermark
    out = [([], [])]
    for sel in (shut, ~shut):
        k, w = keys[sel], wid[sel]
        o = _key_string_order(k, w, w)
        out.append(([(int(a), int(b), 1) for a, b in zip(k[o], w[o])], []))
    return out
