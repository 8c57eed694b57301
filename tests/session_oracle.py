"""CPU restatement of session-window folds on integer microseconds.  TEST INFRASTRUCTURE ONLY.

What the CUDA session fold (``bw_session``, csrc/bw_session.cuh) replaces, restated in plain Python the way
``oracle/pyoracle.py`` restates the sliding windower (paths relative to the bytewax v0.21.1 source tree):

* ``SessionWindower``     -> pysrc/bytewax/operators/windowing.py:671-810 (``_SessionWindowerLogic``)
* ``_session_find_merges``-> windowing.py:688-715
* ``_WindowLogic``        -> windowing.py:1046-1190 (late test, inserts, merge queue, close, notify)
* ``EventClock``          -> windowing.py:230-310 (``oracle.pyoracle.EventClock``)
* accumulators            -> windowing.py:1679-1689 (count_window), :2268-2285 (reduce_window(operator.add)),
                             :2189 / :2236 (max_window / min_window, ``by`` = identity), merged by :1692-1714
* engine                  -> src/operators.rs:755-806 (ascending key string per activation), :808-858 (notify),
                             :862-894 (EOF); session state is never discarded (windowing.py:798-806)

``tools/gen_session_golden.py`` drives the reference's own classes and writes ``tests/golden/session_cases.json``;
``tests/test_oracle_sessions.py`` checks this restatement against it.  Rows are ``[key, window_id, tag, payload]``:
``E`` carries the accumulator, ``L`` the value, ``M`` ``[open_us, close_us, sorted merged ids]``.
"""

from __future__ import annotations

from typing import Dict, List, Optional

from oracle.pyoracle import UTC_MAX_US, UTC_MIN_US, EventClock, key_str

LATE_SESSION_ID = -1  # windowing.py:671
WAIT_FOREVER = (1 << 63) - 1  # BW_WAIT_FOREVER: the watermark never advances on data


def fold_step(reduction: str, acc, v):
    """``acc`` None: a fresh accumulator (builder); the value seeds it (count: ``0 + 1``)."""
    if reduction == "count":
        return 1 if acc is None else acc + 1  # windowing.py:1686
    if acc is None:
        return v  # reduce_window's shim_folder, windowing.py:2268-2276
    if reduction == "sum":
        return acc + v
    if reduction == "max":
        return v if v > acc else acc  # max(acc, v): the first argument wins unless the second is greater
    if reduction == "min":
        return v if v < acc else acc
    raise ValueError(reduction)


def merge_step(reduction: str, into, orig):
    """``into = merger(into, orig)``, windowing.py:1700-1703."""
    if reduction in ("count", "sum"):
        return into + orig
    if reduction == "max":
        return orig if orig > into else into
    if reduction == "min":
        return orig if orig < into else into
    raise ValueError(reduction)


class SessionWindower:
    """``_SessionWindowerLogic``: ``sessions`` is id -> [open, close, merged_ids], dict order == id order."""

    def __init__(self, gap_us: int):
        self.gap = gap_us
        self.max_key = LATE_SESSION_ID
        self.sessions: Dict[int, list] = {}
        self.merge_queue: List[tuple] = []

    def _find_merges(self) -> None:
        # windowing.py:688-729: sort by open (stable: ties keep id order); merge into the running "last"
        if len(self.sessions) < 2:
            return
        order = sorted(self.sessions.items(), key=lambda kv: kv[1][0])
        last_id, last = order.pop(0)
        for this_id, this in order:
            if this[0] - last[1] <= self.gap:
                last[1] = max(last[1], this[1])
                self.merge_queue.append((this_id, last_id))
                last[2].add(this_id)  # direct merges only: this's own merged ids go with it
                del self.sessions[this_id]
            else:
                last_id, last = this_id, this

    def open_for(self, ts: int) -> int:
        # windowing.py:731-762: the FIRST session by id that contains ts or is within gap of it
        for wid, meta in self.sessions.items():
            until_open, since_close = meta[0] - ts, ts - meta[1]
            if until_open <= 0 and since_close <= 0:
                return wid
            if 0 < until_open <= self.gap:
                meta[0] = ts
                self._find_merges()
                return wid
            if 0 < since_close <= self.gap:
                meta[1] = ts
                self._find_merges()
                return wid
        self.max_key += 1
        self.sessions[self.max_key] = [ts, ts, set()]
        return self.max_key

    def merged(self):
        q, self.merge_queue = self.merge_queue, []
        return q

    def close_for(self, watermark: int):
        # windowing.py:774-788: strictly before watermark - gap (UTC_MIN when that is not representable), id order
        close_after = watermark - self.gap
        if close_after < UTC_MIN_US:
            close_after = UTC_MIN_US
        closed = [(wid, meta) for wid, meta in self.sessions.items() if meta[1] < close_after]
        for wid, _ in closed:
            del self.sessions[wid]
        return closed

    def notify_at(self) -> Optional[int]:
        # windowing.py:790-796
        if not self.sessions:
            return None
        return min(m[1] for m in self.sessions.values()) + self.gap


class SessionLogic:
    """``_WindowLogic`` (unordered) over a session windower and a numeric fold."""

    def __init__(self, reduction: str, gap_us: int, wait_us: int, now_us: int):
        self.reduction = reduction
        self.clock = EventClock(wait_us, now_us)
        self.windower = SessionWindower(gap_us)
        self.accs: Dict[int, object] = {}
        self.last_watermark = UTC_MIN_US

    def _flush(self, queue, watermark: int):
        # windowing.py:1064-1108: every insert, then the merge queue, then the close
        for value, ts in queue:
            wid = self.windower.open_for(ts)
            self.accs[wid] = fold_step(self.reduction, self.accs.get(wid), value)
        for orig, targ in self.windower.merged():
            self.accs[targ] = merge_step(self.reduction, self.accs[targ], self.accs.pop(orig))
        events = []
        for wid, meta in self.windower.close_for(watermark):
            events.append((wid, "E", self.accs.pop(wid)))
            events.append((wid, "M", [meta[0], meta[1], sorted(meta[2])]))
        return events

    def on_batch(self, values):
        """``values``: ``(value, ts_us)`` in arrival order (windowing.py:1115-1133)."""
        self.clock.before_batch()
        events, queue = [], []
        watermark = self.last_watermark
        for value, ts in values:
            _, watermark = self.clock.on_item(ts)
            self.last_watermark = watermark
            if ts < watermark:
                events.append((LATE_SESSION_ID, "L", value))
            else:
                queue.append((value, ts))
        return events + self._flush(queue, watermark)

    def on_notify(self):
        watermark = self.clock.on_notify()  # windowing.py:1135-1142
        self.last_watermark = watermark
        return self._flush([], watermark)

    def on_eof(self):
        self.last_watermark = UTC_MAX_US  # windowing.py:1144-1151
        return self._flush([], UTC_MAX_US)


S = 1_000_000
A = 1_640_995_200_000_000  # 2022-01-01T00:00:00Z
F64_VALUES = (1e16, -1e16, 1.0, -1.0, 0.1, 0.2, 0.3, 3.5, -2.25, 1e-3)  # sums whose bits depend on the fold order


def seeded_spec(seed: int) -> dict:
    red = ("count", "sum", "min", "max")[seed % 4]
    dtype = "f64" if (seed // 4) % 2 else "i64"
    gap, wait = (0, S, 2 * S, 5 * S)[(seed // 2) % 4], (0, S, 3 * S, WAIT_FOREVER)[(seed // 3) % 4]
    if gap == 0 and wait == WAIT_FOREVER:  # nothing would ever close or merge: a key would need ~70 sessions
        wait = 3 * S
    return dict(reduction=red, val_dtype=dtype, gap_us=gap, wait_us=wait)


def seeded_steps(seed: int, n_steps: int = 30, n_keys: int = 6, moving: bool = True):
    """A seeded stream of activations and notify steps: keys 1..n_keys plus key 0, timestamps jittered by +-4 s around a
    base that moves forward 1 s per activation, and one item in ten up to 30 s behind (late unless the wait holds the
    watermark back).  ``moving``: the system clock steps forward; otherwise it is frozen and there is no notify step."""
    import random

    rnd = random.Random(9000 + seed)
    spec = seeded_spec(seed)
    now, base, steps = A + 50 * S, A, []
    for _ in range(n_steps):
        if moving:
            now += rnd.randint(0, 3 * S)
        if moving and rnd.random() < 0.25:
            steps.append(["notify", now])
            continue
        n = rnd.randint(1, 25)
        keys = [rnd.randint(0, n_keys) for _ in range(n)]
        ts = [base + rnd.randint(-4 * S, 4 * S) - (rnd.randint(5 * S, 30 * S) if rnd.random() < 0.1 else 0) for _ in range(n)]
        if spec["val_dtype"] == "f64":
            vals = [rnd.choice(F64_VALUES) if rnd.random() < 0.7 else round(rnd.uniform(-100, 100), 3) for _ in range(n)]
        else:
            vals = [rnd.randint(-1000, 1000) for _ in range(n)]
        steps.append(["batch", now, keys, ts, vals])
        base += S
    return spec, steps


SEEDED = range(32)


def run_sessions(spec: dict, steps, eof: bool = True):
    """``spec``: reduction, gap_us, wait_us.  ``steps``: ``["batch", now_us, keys, ts, vals]`` (one activation, with
    ``now_getter() == now_us``) or ``["notify", now_us]`` (the notify phase: every key whose ``notify_at()`` has come,
    src/operators.rs:808-858).  Returns the rows of every step, then of EOF when ``eof``."""
    logics: Dict[str, SessionLogic] = {}
    ids: Dict[str, int] = {}
    acts = []

    def rows_of(ks, events):
        return [[ids[ks], wid, tag, payload] for wid, tag, payload in events]

    for step in steps:
        now = step[1]
        for lg in logics.values():
            lg.clock.now_us = now
        rows = []
        if step[0] == "batch":
            grouped: Dict[str, list] = {}
            for k, t, v in zip(step[2], step[3], step[4]):
                ks = key_str(k)
                ids[ks] = int(k)
                grouped.setdefault(ks, []).append((v, int(t)))
            for ks in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
                lg = logics.get(ks)
                if lg is None:
                    lg = logics[ks] = SessionLogic(spec["reduction"], spec["gap_us"], spec["wait_us"], now)
                rows.extend(rows_of(ks, lg.on_batch(grouped[ks])))
        else:
            for ks in sorted(logics):
                at = logics[ks].windower.notify_at()
                if at is not None and at <= now:
                    rows.extend(rows_of(ks, logics[ks].on_notify()))
        acts.append(rows)
    if eof:
        rows = []
        for ks in sorted(logics):
            rows.extend(rows_of(ks, logics[ks].on_eof()))
        acts.append(rows)
    return acts
