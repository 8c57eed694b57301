"""Streams that take one key of the keyed window kernels to M sessions or windows, and an instrumented run of their CPU
oracles that measures how close each call comes.  TEST INFRASTRUCTURE ONLY.

The kernels K7 (session folds), K8 (``join_window``), K9 (``collect_window``), K10 (session ``join_window``), K11
(``max_window`` / ``min_window`` with ``by=``), K12 (session ``collect_window``), K14 (product ``join_window``) and K16
(product ``join_window`` over sessions) keep a key's state in a fixed array of M <= 64 records, walked by one thread.
What the device counts against M (DESIGN section 10):

* sessions: the records a call holds -- live sessions plus the ones merged away in this call, which keep their slot
  until the call's merges are applied -- and the merged ids the live sessions hold;
* K12 also: the merge intervals the key's sessions hold after the call's merges, before its close (a merge of B into A
  gives A one interval and B's intervals; a chain C -> B -> A gives A two intervals and one merged id);
* windows: the open windows, counting the ones this call opened before its close.

``measure`` runs an oracle with its windowers swapped for subclasses that count these per key and per call, without
changing the oracle.  A test derives what the device must do (rows, or ``BW_ERR_CAPACITY`` at a given step) from
``first_overflow`` of those numbers and M, never from a hand-written expectation.

Builders return a ``(clock, steps)`` pair: ``clock`` has ``gap_us`` (sessions) or ``length_us`` / ``offset_us`` /
``align_us`` (windows), and ``wait_us``; ``steps`` are ``["batch", now_us, keys, ts, vals]`` or ``["notify", now_us]``.
``for_kernel`` turns them into each oracle's step format (handles are running integers).
"""

from __future__ import annotations

import math
import random
from contextlib import contextmanager
from dataclasses import dataclass
from typing import Dict, List, Optional
from unittest import mock

from oracle.pyoracle import SlidingWindower
from tests import arg_window_oracle as aw
from tests import collect_window_oracle as co
from tests import join_window_oracle as jo
from tests import product_join_window_oracle as po
from tests import session_collect_oracle as sc
from tests import session_join_oracle as sj
from tests import session_oracle as so
from tests import session_product_join_oracle as sp

S, A = so.S, so.A
WAIT_FOREVER = so.WAIT_FOREVER
MS = (32, 33, 63, 64)  # around the 32-bit boundary of the u64 masks, and the engine's default of 64


# ---------------------------------------------------------------------------
# instrumentation
# ---------------------------------------------------------------------------


@dataclass
class Call:
    """What one call of one key's logic held at its peak.  Sessions: ``records`` (live plus merged away in this call),
    ``mids`` (merged ids held by live sessions), ``dead`` (largest record index merged away, -1: none), ``merges``,
    ``tie`` (largest record index of the lower of two live sessions with the same open when they were sorted, -1:
    none), ``ivs`` (K12's merge intervals held after the merges, before the close).  Windows: ``open``, ``values``
    (most values played into one window so far), ``wins`` (most windows one value was played into), ``cell`` (largest
    cell, in K9's lowest-free-cell order), ``reuse`` (largest cell given to a new window after a window on it closed in
    an earlier call, -1: none)."""

    step: int
    records: int = 0
    mids: int = 0
    dead: int = -1
    merges: int = 0
    tie: int = -1
    ivs: int = 0
    open: int = 0
    values: int = 0
    wins: int = 0
    cell: int = -1
    reuse: int = -1

    def peak(self, fields=None) -> int:
        """The largest of the numbers a kernel counts against M (``fields``; default: records, merged ids, windows)."""
        return max(getattr(self, f) for f in fields or COUNTED_DEFAULT)


COUNTED_DEFAULT = ("records", "mids", "open")
COUNTED = {"k12": ("records", "mids", "ivs")}  # only K12 keeps merge intervals


def counted(kernel: Optional[str]):
    """The fields of ``Call`` that ``kernel`` counts against M."""
    return COUNTED.get(kernel, COUNTED_DEFAULT)


class _Tracker:
    def __init__(self):
        self.step = 0
        self.logs: List[List[Call]] = []  # per windower (one per key logic), its calls in order

    def steps(self, steps):
        for i, s in enumerate(steps):
            self.step = i
            yield s
        self.step = len(steps)  # EOF


_active: Optional[_Tracker] = None


class _Ids(set):
    """A session's merged ids; ``add`` runs in ``_find_merges`` while the merged-away session is still in the dict."""

    def __init__(self, owner):
        super().__init__()
        self.owner = owner

    def add(self, x):
        super().add(x)
        w = self.owner
        held = sum(len(m[2]) for m in w.sessions.values()) - len(w.sessions[x][2])  # its own ids go with it
        c = w._call()
        c.mids = max(c.mids, held)


class TrackedSessions(so.SessionWindower):
    def __init__(self, gap_us: int):
        super().__init__(gap_us)
        self.calls: List[Call] = []
        self._cur: Optional[Call] = None
        self._rec: List[int] = []  # record order on the device: live sessions in id order, then the call's new ones
        self._ivs: Dict[int, int] = {}  # live session id -> its merge intervals (K12)
        _active.logs.append(self.calls)

    def _call(self) -> Call:
        if self._cur is None:
            self._cur = Call(_active.step, records=len(self._rec), mids=sum(len(m[2]) for m in self.sessions.values()),
                             ivs=sum(self._ivs.values()))
        return self._cur

    def _find_merges(self) -> None:
        c = self._call()
        by_open = {}
        for wid, m in self.sessions.items():
            by_open.setdefault(m[0], []).append(self._rec.index(wid))
        for ix in by_open.values():
            if len(ix) > 1:
                c.tie = max(c.tie, min(ix))
        super()._find_merges()

    def open_for(self, ts: int) -> int:
        c = self._call()
        q0, top = len(self.merge_queue), self.max_key
        wid = super().open_for(ts)
        if self.max_key != top:
            self._rec.append(wid)
            self.sessions[wid][2] = _Ids(self)
        for orig, _into in self.merge_queue[q0:]:
            c.merges += 1
            c.dead = max(c.dead, self._rec.index(orig))
        c.records = max(c.records, len(self._rec))
        return wid

    def merged(self):
        """The merge queue, in the order the logic applies it: ``into`` takes one interval and ``orig``'s."""
        q = super().merged()
        for orig, into in q:
            self._ivs[into] = self._ivs.get(into, 0) + 1 + self._ivs.pop(orig, 0)
        c = self._call()
        c.ivs = max(c.ivs, sum(self._ivs.values()))
        return q

    def close_for(self, watermark: int):
        closed = super().close_for(watermark)
        for wid, _ in closed:  # a closing session's intervals go with it
            self._ivs.pop(wid, None)
        self.calls.append(self._call())
        self._cur = None
        self._rec = list(self.sessions)
        return closed


class TrackedWindows(SlidingWindower):
    def __init__(self, length_us: int, offset_us: int, align_us: int):
        super().__init__(length_us, offset_us, align_us)
        self.calls: List[Call] = []
        self._cur: Optional[Call] = None
        self._cells, self._freed, self._count = {}, set(), {}
        _active.logs.append(self.calls)

    def _call(self) -> Call:
        if self._cur is None:
            self._cur = Call(_active.step, open=len(self.opened))
        return self._cur

    def open_for(self, ts: int):
        c = self._call()
        new = [w for w in self.intersects(ts) if w not in self.opened]
        ids = super().open_for(ts)
        for wid in new:  # (ascending id, as the device opens them)
            used = set(self._cells.values())
            cell = next(i for i in range(len(used) + 1) if i not in used)
            self._cells[wid] = cell
            c.cell = max(c.cell, cell)
            if cell in self._freed:
                c.reuse = max(c.reuse, cell)
        for wid in ids:
            self._count[wid] = self._count.get(wid, 0) + 1
            c.values = max(c.values, self._count[wid])
        c.wins = max(c.wins, len(ids))
        c.open = max(c.open, len(self.opened))
        return ids

    def close_for(self, watermark: int):
        closed = super().close_for(watermark)
        for wid, _ in closed:
            self._freed.add(self._cells.pop(wid))
            self._count.pop(wid, None)
        self.calls.append(self._call())
        self._cur = None
        return closed


RUNNERS = {"k7": so.run_sessions, "k8": jo.run_join_window, "k9": co.run_collect_window, "k10": sj.run_session_join,
           "k11": aw.run_arg_window, "k12": sc.run_session_collect, "k14": po.run_product_join_window,
           "k16": sp.run_session_product_join}


@contextmanager
def _instrumented():
    global _active
    tr = _Tracker()
    _active = tr
    try:
        # (K12's oracle imports the class by name; K14 and K16 reach theirs through K8's and K10's logic)
        with mock.patch.object(so, "SessionWindower", TrackedSessions), mock.patch.object(sj, "SessionWindower", TrackedSessions), \
                mock.patch.object(sc, "SessionWindower", TrackedSessions), mock.patch.object(jo, "SlidingWindower", TrackedWindows):
            yield tr
    finally:
        _active = None


def measure(kernel: str, spec: dict, steps):
    """The oracle of ``kernel`` over ``steps`` (its own format), instrumented: ``(its result, logs)``, where ``logs`` has
    one list of ``Call`` per key logic."""
    with _instrumented() as tr:
        out = RUNNERS[kernel](spec, tr.steps(steps))
    return out, tr.logs


def calls(logs) -> List[Call]:
    return [c for log in logs for c in log]


def peak(logs, field: str) -> int:
    return max((getattr(c, field) for c in calls(logs)), default=-1)


def first_overflow(logs, M: int, kernel: Optional[str] = None) -> Optional[int]:
    """The first step (``len(steps)``: EOF) in which a key needs more than M of what ``kernel`` counts: records, merged
    ids or open windows, and for K12 merge intervals."""
    fields = counted(kernel)
    return min((c.step for c in calls(logs) if c.peak(fields) > M), default=None)


# ---------------------------------------------------------------------------
# values
# ---------------------------------------------------------------------------

F64_SPECIAL = (0.0, -0.0, math.nan, math.inf, -math.inf)
I64_BIG = (1 << 62) + 12345  # sums of a few of these wrap past 2^63


def values(rnd: random.Random, n: int, dtype: str) -> list:
    """f64: ``session_oracle.F64_VALUES`` (fold order shows in the bits) with a few signed zeros, NaN and infinities;
    i64: small values and ones near +-2^62, so that sums wrap."""
    if dtype == "f64":
        return [rnd.choice(F64_SPECIAL) if rnd.random() < 0.06 else rnd.choice(so.F64_VALUES) for _ in range(n)]
    return [rnd.choice((I64_BIG, -I64_BIG, I64_BIG + 7)) if rnd.random() < 0.4 else rnd.randint(-1000, 1000) for _ in range(n)]


def revalue(steps, dtype: str, seed: int):
    """The same steps with values drawn afresh as ``dtype``."""
    rnd = random.Random(seed)
    return [s if s[0] != "batch" else s[:4] + [values(rnd, len(s[2]), dtype)] for s in steps]


def _batch(rnd, now, items, dtype, key=7):
    """items: (ts, key or None) in arrival order."""
    keys = [key if k is None else k for _, k in items]
    return ["batch", now, keys, [t for t, _ in items], values(rnd, len(items), dtype)]


# ---------------------------------------------------------------------------
# session builders (one hot key 7, next to a light key 3 that keeps the grid honest)
# ---------------------------------------------------------------------------

G = S  # the gap of the gapped builders; sessions 2 G apart stay apart, a bridge at +G joins two


def fill(M: int, seed: int, n: Optional[int] = None, gap: int = G, calls_: int = 1, dtype: str = "f64"):
    """One key opens n (default M) sessions, wait forever, in one call or spread over ``calls_``; arrival order
    seeded.  Each session gets one to three values at its one timestamp."""
    rnd = random.Random(seed)
    n = M if n is None else n
    d = 3 * gap if gap else S
    slots = list(range(n))
    rnd.shuffle(slots)
    items = [(A + p * d, None) for p in slots for _ in range(rnd.randint(1, 3))]
    items.insert(rnd.randrange(len(items)), (A, 3))
    per = -(-len(items) // calls_)
    steps = [_batch(rnd, A, items[i : i + per], dtype) for i in range(0, len(items), per)]
    return dict(gap_us=gap, wait_us=WAIT_FOREVER), steps


ORDERS = ("asc", "desc", "middle", "random")


def collapse(M: int, seed: int, order: str = "asc", extra: int = 0, dtype: str = "f64"):
    """M sessions 2 G apart in one call (ids in position order), then one call whose M - 1 bridges (each G after a
    session) join them all into session 0: M - 1 merges in one call, in ``order``.  Then ``extra`` calls, each opening a
    session beyond the survivor and bridging it in: one more merged id each."""
    rnd = random.Random(seed)
    t = [A + 2 * G * p for p in range(M)]
    steps = [_batch(rnd, A, [(x, None) for x in t] + [(A, 3)], dtype)]
    bridges = list(range(M - 1))
    if order == "desc":
        bridges.reverse()
    elif order == "middle":
        mid = (M - 1) // 2
        bridges = sorted(bridges, key=lambda p: (abs(p - mid), p))
    elif order == "random":
        rnd.shuffle(bridges)
    steps.append(_batch(rnd, A, [(t[p] + G, None) for p in bridges], dtype))
    close = t[-1]
    for e in range(extra):
        steps.append(_batch(rnd, A, [(close + 2 * G, None), (close + G, None)], dtype))
        close += 2 * G
    return dict(gap_us=G, wait_us=WAIT_FOREVER), steps


def records_not_live(M: int, seed: int, below: bool = False, dtype: str = "f64"):
    """n = M (``below``: M - 1) sessions; then one call that merges session 1 into 0 and opens a new session.  With
    n = M the call holds M records (M - 1 live, one merged away) before the new session, which makes M + 1."""
    rnd = random.Random(seed)
    n = M - 1 if below else M
    t = [A + 2 * G * p for p in range(n)]
    steps = [_batch(rnd, A, [(x, None) for x in t], dtype),
             _batch(rnd, A, [(t[0] + G, None), (t[-1] + 10 * G, None), (A, 3)], dtype)]
    return dict(gap_us=G, wait_us=WAIT_FOREVER), steps


def many_keys(M: int, seed: int, n_keys: int = 300, dtype: str = "f64"):
    """n_keys keys, each with M - 31 .. M sessions 2 G apart (33 .. 64 at M = 64), wait 2 G M.  Then a call of bridges
    (merges) and late rows, notify steps of a moving clock that close the oldest sessions in slices, a call that opens
    new sessions in their place, and EOF."""
    rnd = random.Random(seed)
    wait = 2 * G * M  # nothing closes in the first call
    per_key = {k: rnd.randint(max(1, M - 31), M) for k in range(1, n_keys + 1)}
    t0 = {k: A + rnd.randrange(0, 4) * G for k in per_key}
    first = [(t0[k] + 2 * G * p, k) for k, n in per_key.items() for p in range(n) for _ in range(rnd.randint(1, 2))]
    rnd.shuffle(first)
    now = A
    steps = [_batch(rnd, now, first, dtype)]
    second = []
    for k, n in per_key.items():
        for p in rnd.sample(range(n - 1), min(n - 1, rnd.randint(0, 6))):
            second.append((t0[k] + 2 * G * p + G, k))  # extends p's close to within gap of p + 1: a merge
        if rnd.random() < 0.3:
            second.append((A - wait - 10 * S, k))  # late
    rnd.shuffle(second)
    now += S
    steps.append(_batch(rnd, now, second, dtype))
    for _ in range(3):  # the watermark moves with the system clock: each notify closes the next ~10 sessions
        now += 30 * S
        steps.append(["notify", now])
    third = []
    for k, n in per_key.items():
        for p in range(rnd.randint(0, 9) if n <= M - 10 else 0):  # (a full key only extends its last session)
            third.append((t0[k] + 2 * G * (n + 2 + p), k))
        third.append((t0[k] + 2 * G * (n - 1) + G // 2, k))
        if rnd.random() < 0.2:
            third.append((A - wait - 10 * S, k))  # late
    rnd.shuffle(third)
    now += S
    steps.append(_batch(rnd, now, third, dtype))
    return dict(gap_us=G, wait_us=wait), steps


def session_builders(M: int):
    """name -> (clock, steps) for every session builder at M."""
    out = {
        "fill_one_call": fill(M, 1),
        "fill_gap0": fill(M, 2, gap=0),
        "fill_spread": fill(M, 3, calls_=4),
        "fill_over": fill(M, 4, n=M + 1),
        "fill_over_spread": fill(M, 5, n=M + 1, calls_=3, gap=0),
        "collapse_extra1": collapse(M, 10, "asc", extra=1),
        "collapse_extra2": collapse(M, 11, "asc", extra=2),
        # a descending chain leaves one merged id but M - 1 intervals: K12's interval limit alone
        "collapse_desc_extra1": collapse(M, 16, "desc", extra=1),
        "collapse_desc_extra2": collapse(M, 17, "desc", extra=2),
        "records_not_live": records_not_live(M, 20),
        "records_not_live_below": records_not_live(M, 21, below=True),
        "many_keys": many_keys(M, 30),
    }
    for i, o in enumerate(ORDERS):
        out[f"collapse_{o}"] = collapse(M, 12 + i, o)
    return out


SESSION_BUILDERS = sorted(session_builders(4))


# ---------------------------------------------------------------------------
# window builders
# ---------------------------------------------------------------------------

L = 10 * S  # tumbling length


def tumbling(M: int, seed: int, n: Optional[int] = None, order: str = "desc", reopen: int = 0):
    """One key opens n (default M) tumbling windows in one call, in descending or random id order (wait long enough
    that none is late).  Notify steps of a moving clock then close them in slices of 8, oldest first.  ``reopen``:
    after the first slice closes, a call opens that many new windows (ids n, n + 1, ...), which take the cells the
    closed windows left -- in descending order those are the highest cells -- and a light key 3 comes and goes."""
    rnd = random.Random(seed)
    n = M if n is None else n
    wait = (n + 2) * L
    ids = list(range(n))[::-1]
    if order == "random":
        rnd.shuffle(ids)
    items = [(A + w * L + rnd.randrange(L), None) for w in ids for _ in range(rnd.randint(1, 2))]
    items.insert(rnd.randrange(len(items)), (A + 5 * S, 3))
    now = A + n * L
    steps = [_batch(rnd, now, items, "i64")]
    closed = 0
    while closed < n + reopen:
        now += 8 * L
        steps.append(["notify", now])
        closed += 8
        if reopen and len(steps) == 2:
            lo = n
            steps.append(_batch(rnd, now, [(A + (lo + j) * L + rnd.randrange(L), None) for j in range(reopen)]
                                + [(A + (lo + 1) * L, 3), (A - 5 * L, None)], "i64"))
    return dict(length_us=L, offset_us=L, align_us=A, wait_us=wait), steps


O = 2 * S  # sliding offset


def sliding(M: int, seed: int, k: Optional[int] = None, more: bool = True):
    """Sliding windows of length k * O (default M * O), offset O: every item is in k windows.  A call of items in one
    offset bucket opens k windows; then (``more``) a moving clock closes 4 of them and a call in the bucket 4 later
    opens 4 new ones, and a light key 3 rides along.  k = M + 1 needs M + 1 windows on its first item."""
    rnd = random.Random(seed)
    k = M if k is None else k
    b0 = 100
    now = A + b0 * O
    xs = sorted(rnd.randrange(O // 2) for _ in range(6))
    steps = [_batch(rnd, now, [(A + b0 * O + x, None) for x in xs] + [(A + b0 * O, 3)], "i64")]
    if more:
        now += 4 * O
        steps.append(["notify", now])
        wm = A + b0 * O + xs[-1] + 4 * O
        steps.append(_batch(rnd, now, [(wm + j, None) for j in range(3)] + [(wm - 3 * O, None)], "i64"))
    return dict(length_us=k * O, offset_us=O, align_us=A, wait_us=0), steps


def sliding_creep(M: int, seed: int, n_calls: int = 9):
    """Sliding windows of length M * O, offset O: every item is in M windows.  The first call puts one to three items in
    one offset bucket, which opens M windows; each later call is a notify whose moving clock takes the watermark to the
    next bucket's start, closing the lowest window, then one to three items in that bucket, which open one window on
    the cell the closed one left.  The items of a call share one timestamp, and the system clock runs O ahead of it
    (so the notify wakes the key, and with wait 0 nothing is late).  So a window's side lists fill over several calls,
    and windows opened in different calls hold different generations: under ``complete`` a clear frees a value in some
    of its windows while others still hold it, and the value is released only when the last of them clears or
    closes."""
    rnd = random.Random(seed)
    b, steps = 100, []
    for i in range(n_calls):
        x = rnd.randrange(O // 2)
        if i:
            b += 1
            steps.append(["notify", A + b * O + O])  # watermark: the last items' ts + (now - their arrival) = A + b O
        items = [(A + b * O + x, None)] * rnd.randint(1, 3) + ([(A + b * O, 3)] if i == 0 else [])
        steps.append(_batch(rnd, A + b * O + x + O, items, "i64"))
    return dict(length_us=M * O, offset_us=O, align_us=A, wait_us=0), steps


def window_builders(M: int):
    return {
        "tumbling_desc": tumbling(M, 40),
        "tumbling_random": tumbling(M, 41, order="random"),
        "tumbling_over": tumbling(M, 42, n=M + 1),
        "tumbling_reopen": tumbling(M, 43, reopen=5),
        "sliding_full": sliding(M, 50),
        "sliding_over": sliding(M, 51, k=M + 1),
        "sliding_creep": sliding_creep(M, 53),
        "many_keys": window_many_keys(M, 52),
    }


def window_many_keys(M: int, seed: int, n_keys: int = 300):
    """n_keys keys, each opening M - 31 .. M tumbling windows in one call in random order, then a moving clock closing
    them in slices, with late rows."""
    rnd = random.Random(seed)
    per_key = {k: rnd.randint(max(1, M - 31), M) for k in range(1, n_keys + 1)}
    wait = (M + 2) * L
    items = [(A + w * L + rnd.randrange(L), k) for k, n in per_key.items() for w in range(n)]
    rnd.shuffle(items)
    now = A + M * L
    steps = [_batch(rnd, now, items, "i64")]
    for _ in range(3):
        now += 16 * L
        late = [(A + rnd.randrange(4) * L, k) for k in rnd.sample(sorted(per_key), 40)]
        steps.append(["notify", now])
        steps.append(_batch(rnd, now, late, "i64"))
    return dict(length_us=L, offset_us=L, align_us=A, wait_us=wait), steps


WINDOW_BUILDERS = sorted(window_builders(4))


# ---------------------------------------------------------------------------
# one stream, every kernel's step format
# ---------------------------------------------------------------------------


def for_kernel(kernel: str, clock: dict, steps, **spec):
    """``(spec, steps)`` in ``kernel``'s oracle format.  K7 takes the values; the others take running handles (K8, K10,
    K14, K16: side = handle mod sides; K11: the value is the by-value; K12: no side).  ``spec`` adds the kernel's own
    fields."""
    spec = dict(clock, **spec)
    if kernel == "k7":
        return spec, [list(s) for s in steps]
    out, nxt = [], 0
    for s in steps:
        if s[0] != "batch":
            out.append(list(s))
            continue
        n = len(s[2])
        hs = list(range(nxt, nxt + n))
        nxt += n
        if kernel == "k12":
            out.append(["batch", s[1], s[2], s[3], hs])
        elif kernel == "k11":
            out.append(["batch", s[1], s[2], s[3], [aw.enc(v) for v in s[4]], hs])
        else:
            out.append(["batch", s[1], s[2], s[3], [h % spec.get("sides", 1) for h in hs], hs])
    return spec, out
