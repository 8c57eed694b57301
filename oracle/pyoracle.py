"""CPU oracle for the windowed-fold hot path.  TEST INFRASTRUCTURE ONLY.

This module is a plain-Python restatement, on integer microseconds, of the
part of the reference (bytewax v0.21.1) that the CUDA path replaces.  It is
imported only by ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs, and only as the checker.  The
product path (``bytewax_b200``) never imports anything under ``oracle/``.

Parity status: **pinned**.  ``oracle/gen_golden.py`` drives the reference's
own, unmodified ``_WindowLogic`` / ``_EventClockLogic`` /
``_SlidingWindowerLogic`` (imported in place from ``$BYTEWAX_SRC/pysrc``)
and commits the resulting vectors under ``tests/golden/``;
``tests/test_oracle_golden.py`` checks this restatement against them and
against the expected lists of the reference's own tests.

What each piece follows (paths relative to the bytewax v0.21.1 source tree):

* ``EventClock``      -> pysrc/bytewax/operators/windowing.py:230-310
* ``SlidingWindower`` -> pysrc/bytewax/operators/windowing.py:603-668
  (tumbling = sliding with offset == length, windowing.py:921-926)
* ``WindowLogic``     -> pysrc/bytewax/operators/windowing.py:1046-1190
* fold accumulators   -> windowing.py:1692-1714 (_FoldWindowLogic),
  :1679-1689 (count_window), :2268-2285 (reduce_window),
  :2189/:2236 (max_window / min_window)
* ``StatefulBatchEngine`` -> src/operators.rs:755-806 (on_batch per key in
  ascending key-string order), :862-894 (on_eof), :796-799 (discard)

All times are int microseconds since the Unix epoch.  Python ints are
unbounded, so the reference's ``OverflowError`` branches
(windowing.py:271-285) are restated as explicit range checks.
"""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence, Tuple

# windowing.py:58-62 -- datetime.min / datetime.max in UTC, as integer us.
UTC_MIN_US = -62_135_596_800_000_000
UTC_MAX_US = 253_402_300_799_999_999


def splitmix64(x: int) -> int:
    """SURVEY.md section 8(d) input generator."""
    x = (x + 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
    z = x
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return z ^ (z >> 31)


# ---------------------------------------------------------------------------
# Clock (windowing.py:230-310)
# ---------------------------------------------------------------------------


@dataclass
class EventClock:
    """Restates ``_EventClockLogic``.

    ``now_us`` is what ``now_getter()`` returns; parity runs freeze it
    (SURVEY.md section 7 "System time leaks into results").
    """

    wait_us: int
    now_us: int = 0
    watermark_base: int = UTC_MIN_US
    system_time_of_max_event: Optional[int] = None
    _system_now: int = field(init=False, default=0)

    def __post_init__(self) -> None:
        # windowing.py:245-248
        self._system_now = self.now_us
        if self.system_time_of_max_event is None:
            self.system_time_of_max_event = self._system_now

    def before_batch(self) -> None:
        # windowing.py:250-261: never let "now" go backwards.
        if self.now_us > self._system_now:
            self._system_now = self.now_us

    def _watermark(self) -> int:
        wm = self.watermark_base + (self._system_now - self.system_time_of_max_event)
        return wm

    def on_item(self, ts: int) -> Tuple[int, int]:
        # windowing.py:263-287
        watermark = self._watermark()
        cand = ts - self.wait_us
        # datetime arithmetic raises OverflowError below datetime.min
        # (windowing.py:281-285): the candidate is then ignored.
        if cand >= UTC_MIN_US and cand > watermark:
            self.watermark_base = cand
            self.system_time_of_max_event = self._system_now
            return ts, cand
        return ts, watermark

    def on_notify(self) -> int:
        # windowing.py:289-298
        self.before_batch()
        return self._watermark()

    def on_eof(self) -> int:
        # windowing.py:300-302
        return UTC_MAX_US


# ---------------------------------------------------------------------------
# Windower (windowing.py:603-668)
# ---------------------------------------------------------------------------


@dataclass
class SlidingWindower:
    length_us: int
    offset_us: int
    align_us: int
    # window_id -> (open_us, close_us); dict order == first-opened order
    opened: Dict[int, Tuple[int, int]] = field(default_factory=dict)

    def intersects(self, ts: int) -> List[int]:
        # windowing.py:611-618; Python // floors toward -inf.
        since = ts - self.align_us
        return list(
            range((since - self.length_us) // self.offset_us + 1, since // self.offset_us + 1)
        )

    def metadata_for(self, wid: int) -> Tuple[int, int]:
        # windowing.py:620-623
        open_us = self.align_us + self.offset_us * wid
        return (open_us, open_us + self.length_us)

    def open_for(self, ts: int) -> List[int]:
        # windowing.py:626-633
        ids = self.intersects(ts)
        for wid in ids:
            if wid not in self.opened:
                self.opened[wid] = self.metadata_for(wid)
        return ids

    def late_for(self, ts: int) -> List[int]:
        # windowing.py:636-637
        return self.intersects(ts)

    def close_for(self, watermark: int) -> List[Tuple[int, Tuple[int, int]]]:
        # windowing.py:645-654: first-opened order, close_time <= watermark.
        closed = [(wid, meta) for wid, meta in self.opened.items() if meta[1] <= watermark]
        for wid, _ in closed:
            del self.opened[wid]
        return closed

    def is_empty(self) -> bool:
        return len(self.opened) <= 0


# ---------------------------------------------------------------------------
# Fold accumulators (windowing.py:1692-1714 and the composites above it)
# ---------------------------------------------------------------------------

REDUCTIONS = ("count", "sum", "min", "max", "mean")


def _fold_builder(reduction: str) -> Callable[[], Any]:
    if reduction == "count":
        return lambda: 0  # windowing.py:1685
    if reduction == "mean":
        return lambda: (0.0, 0)  # fold_window with a (sum, count) accumulator
    return lambda: None  # reduce_window seeds with None, windowing.py:2268-2274


def _fold_step(reduction: str) -> Callable[[Any, Any], Any]:
    if reduction == "count":
        return lambda s, _v: s + 1  # windowing.py:1686
    if reduction == "sum":
        return lambda s, v: v if s is None else s + v
    if reduction == "min":
        # min(s, v) keeps the first extremal value on ties, windowing.py:2236
        return lambda s, v: v if s is None else min(s, v)
    if reduction == "max":
        return lambda s, v: v if s is None else max(s, v)
    if reduction == "mean":
        return lambda s, v: (s[0] + float(v), s[1] + 1)
    raise ValueError(reduction)


# ---------------------------------------------------------------------------
# _WindowLogic (windowing.py:1046-1190)
# ---------------------------------------------------------------------------


@dataclass
class WindowLogic:
    clock: EventClock
    windower: SlidingWindower
    reduction: str
    ordered: bool
    accs: Dict[int, Any] = field(default_factory=dict)
    queue: List[Tuple[Any, int]] = field(default_factory=list)
    last_watermark: int = UTC_MIN_US

    def _flush(self, watermark: int) -> List[Tuple[int, str, Any]]:
        # windowing.py:1095-1108
        if self.ordered:
            due = [e for e in self.queue if e[1] <= watermark]
            self.queue = [e for e in self.queue if not (e[1] <= watermark)]
            due.sort(key=lambda e: e[1])  # stable, windowing.py:1101
        else:
            due = self.queue
            self.queue = []
        step = _fold_step(self.reduction)
        build = _fold_builder(self.reduction)
        # _handle_inserts, windowing.py:1064-1077 (fold emits nothing on value)
        for value, ts in due:
            for wid in self.windower.open_for(ts):
                if wid not in self.accs:
                    self.accs[wid] = build()
                self.accs[wid] = step(self.accs[wid], value)
        # _handle_merged: sliding windows never merge (windowing.py:640-642)
        # _handle_closed, windowing.py:1087-1093: "E" then "M" per window
        events: List[Tuple[int, str, Any]] = []
        for wid, meta in self.windower.close_for(watermark):
            acc = self.accs.pop(wid)
            events.append((wid, "E", acc))
            events.append((wid, "M", meta))
        return events

    def is_empty(self) -> bool:
        # windowing.py:1110-1113
        return len(self.accs) <= 0 and len(self.queue) <= 0 and self.windower.is_empty()

    def on_batch(self, values: Sequence[Tuple[Any, int]]) -> Tuple[List[Tuple[int, str, Any]], bool]:
        """``values`` are ``(value, ts_us)`` in arrival order."""
        # windowing.py:1115-1133
        self.clock.before_batch()
        events: List[Tuple[int, str, Any]] = []
        watermark = self.last_watermark
        for value, ts in values:
            _, watermark = self.clock.on_item(ts)
            assert watermark >= self.last_watermark
            self.last_watermark = watermark
            if ts < watermark:
                events.extend((wid, "L", value) for wid in self.windower.late_for(ts))
            else:
                self.queue.append((value, ts))
        events.extend(self._flush(watermark))
        return events, self.is_empty()

    def on_notify(self) -> Tuple[List[Tuple[int, str, Any]], bool]:
        # windowing.py:1135-1142
        watermark = self.clock.on_notify()
        assert watermark >= self.last_watermark
        self.last_watermark = watermark
        return self._flush(watermark), self.is_empty()

    def notify_at(self) -> Optional[int]:
        # windowing.py:1153-1180 with `to_system_utc` == identity (the EventClock default, windowing.py:407):
        # the earliest close time of an opened window; in ordered mode also the head of the queue
        at = min((meta[1] for meta in self.windower.opened.values()), default=None)
        if self.ordered and self.queue:
            q = self.queue[0][1]
            at = q if at is None else min(at, q)
        return at

    def on_eof(self) -> Tuple[List[Tuple[int, str, Any]], bool]:
        # windowing.py:1144-1151
        watermark = self.clock.on_eof()
        self.last_watermark = watermark
        return self._flush(watermark), self.is_empty()


# ---------------------------------------------------------------------------
# The engine half: StatefulBatchOp (src/operators.rs:549-1038)
# ---------------------------------------------------------------------------


@dataclass
class FoldSpec:
    """Configuration of one windowed fold; mirrors ``bw_fold_spec`` in include/bwgpu.h."""

    reduction: str = "count"
    length_us: int = 60_000_000
    offset_us: Optional[int] = None  # None -> tumbling (offset == length)
    align_us: int = 1_640_995_200_000_000  # 2022-01-01T00:00:00Z, benchmark_windowing.py:14
    wait_us: int = 0
    ordered: bool = False
    now_us: int = 0  # frozen now_getter

    def __post_init__(self) -> None:
        if self.offset_us is None:
            self.offset_us = self.length_us
        assert self.reduction in REDUCTIONS
        assert 0 < self.offset_us <= self.length_us  # windowing.py:880-883


def key_str(key: int) -> str:
    """Canonical u64 -> ``str`` key mapping at the API boundary (SURVEY.md section 7)."""
    return str(int(key))


class StatefulBatchEngine:
    """One worker's ``stateful_batch`` step driving ``WindowLogic`` per key.

    ``on_batch`` == one activation with one epoch's items
    (src/operators.rs:755-806); ``on_eof`` == src/operators.rs:862-894.
    Output rows are ``(key, window_id, tag, payload)`` in the order the
    reference gives them downstream.
    """

    def __init__(self, spec: FoldSpec):
        self.spec = spec
        self.logics: Dict[str, WindowLogic] = {}
        self._keys: Dict[str, int] = {}
        self.now_us = spec.now_us
        self.sched: Dict[str, int] = {}  # key -> system time of its next notification (src/operators.rs:645-650)

    def set_now(self, now_us: int) -> None:
        """What ``now_getter()`` returns from here on (every logic samples it in ``before_batch`` / ``on_notify``)."""
        self.now_us = now_us
        for logic in self.logics.values():
            logic.clock.now_us = now_us

    def on_notify(self, now_us: int):
        """The notify phase at system time ``now_us`` (src/operators.rs:808-858): every key whose scheduled time has come,
        in ascending key-string order."""
        self.set_now(now_us)
        out = []
        for ks in sorted(k for k, at in self.sched.items() if at <= now_us):
            logic = self.logics[ks]
            events, done = logic.on_notify()
            out.extend((self._keys[ks], wid, tag, payload) for wid, tag, payload in events)
            self._resched(ks, logic, done)
        return out

    def _resched(self, ks: str, logic, done: bool) -> None:
        if done:
            del self.logics[ks]  # src/operators.rs:796-799
            self.sched.pop(ks, None)
            return
        at = logic.notify_at()
        if at is None:
            self.sched.pop(ks, None)
        else:
            self.sched[ks] = at

    def _build(self) -> WindowLogic:
        s = self.spec
        return WindowLogic(
            EventClock(s.wait_us, self.now_us),
            SlidingWindower(s.length_us, s.offset_us, s.align_us),
            s.reduction,
            s.ordered,
        )

    def on_batch(self, keys: Iterable[int], ts: Iterable[int], vals: Iterable[Any]):
        grouped: Dict[str, List[Tuple[Any, int]]] = {}
        for k, t, v in zip(keys, ts, vals):
            ks = key_str(k)
            self._keys[ks] = int(k)
            grouped.setdefault(ks, []).append((v, int(t)))
        out = []
        # BTreeMap<StateKey, _> iteration == ascending key *string* order
        # (src/operators.rs:758-767).
        for ks in sorted(grouped):
            logic = self.logics.get(ks)
            if logic is None:
                logic = self.logics[ks] = self._build()
            events, done = logic.on_batch(grouped[ks])
            k = self._keys[ks]
            out.extend((k, wid, tag, payload) for wid, tag, payload in events)
            self._resched(ks, logic, done)
        return out

    def on_eof(self):
        out = []
        for ks in sorted(self.logics):  # src/operators.rs:866
            events, done = self.logics[ks].on_eof()
            k = self._keys[ks]
            out.extend((k, wid, tag, payload) for wid, tag, payload in events)
            if done:
                del self.logics[ks]
        return out


def split_streams(rows):
    """``window()``'s three ``filter_map_value`` passes (windowing.py:1321-1338)."""
    down = [(k, (wid, p)) for k, wid, tag, p in rows if tag == "E"]
    late = [(k, (wid, p)) for k, wid, tag, p in rows if tag == "L"]
    meta = [(k, (wid, p)) for k, wid, tag, p in rows if tag == "M"]
    return down, late, meta


def run_fold(spec: FoldSpec, batches, eof: bool = True):
    """Run batches ``[(keys, ts, vals), ...]``; returns per-activation row lists."""
    eng = StatefulBatchEngine(spec)
    acts = [eng.on_batch(k, t, v) for k, t, v in batches]
    if eof:
        acts.append(eng.on_eof())
    return acts


def dest_rank(key: int, world: int) -> int:
    """Routing of a key to its owning rank.

    The reference routes with Rust's SipHash-1-3 ``DefaultHasher``
    (src/operators.rs:567-568, src/timely.rs:455-465) which is un-vendored and
    un-pinned by any reference test (SURVEY.md section 8c): any deterministic
    hash is conformant.  This is the one ``bytewax_b200`` uses
    (``bw_route`` in include/bwgpu.h): high 32 bits of mix64(key), scaled.
    """
    h = mix64(key)
    return ((h >> 32) * world) >> 32


def mix64(x: int) -> int:
    """splitmix64 finaliser without the increment (== csrc ``bw_mix64``)."""
    z = x & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return z ^ (z >> 31)


# ---------------------------------------------------------------------------
# Synthetic inputs of SURVEY.md section 8(d)
# ---------------------------------------------------------------------------


def c1_rows(start: int, n: int, n_keys: int = 1_000_000, align_us: int = 1_640_995_200_000_000):
    """Config C1: key_i = splitmix64(0x5EED ^ i) mod n_keys; val_i = i; ts_i = align + i us."""
    keys = [splitmix64(0x5EED ^ i) % n_keys for i in range(start, start + n)]
    vals = list(range(start, start + n))
    ts = [align_us + i for i in range(start, start + n)]
    return keys, ts, vals


# ---------------------------------------------------------------------------
# Config C2: stateful_map with the anomaly detector of examples/anomaly_detector.py:16-48
# (engine half: operators/__init__.py:1024-1042 `_StatefulLogic.on_batch`, :2860-2890)
# ---------------------------------------------------------------------------


class ZScoreDetector:
    """Per-key state of the reference's example mapper, restated verbatim in behaviour:
    last-N values newest first, ``mu = sum/len``, ``sigma = (sum((v-mu)**2)/len) ** 0.5`` (both
    summed newest -> oldest like Python's ``sum``), anomalous iff ``mu and sigma`` are truthy and
    ``abs(v - mu) / sigma > threshold`` evaluated BEFORE the push (anomaly_detector.py:33-46)."""

    def __init__(self, window: int = 10, threshold: float = 2.0):
        self.window, self.threshold = window, threshold
        self.last: List[float] = []
        self.mu: Optional[float] = None
        self.sigma: Optional[float] = None

    def on_value(self, value: float):
        anomalous = False
        if self.mu and self.sigma:
            anomalous = abs(value - self.mu) / self.sigma > self.threshold
        self.last.insert(0, value)
        del self.last[self.window:]
        n = len(self.last)
        self.mu = sum(self.last) / n
        self.sigma = (sum((v - self.mu) ** 2 for v in self.last) / n) ** 0.5
        return (value, self.mu, self.sigma, anomalous)


def run_zscore(batches, window: int = 10, threshold: float = 2.0):
    """``batches`` = [(keys, vals), ...] -> per batch a list of (mu, sigma, anomalous) aligned with the input rows."""
    states: Dict[int, ZScoreDetector] = {}
    out = []
    for keys, vals in batches:
        rows = []
        for k, v in zip(keys, vals):
            st = states.get(int(k))
            if st is None:
                st = states[int(k)] = ZScoreDetector(window, threshold)
            _, mu, sigma, flag = st.on_value(float(v))
            rows.append((mu, sigma, flag))
        out.append(rows)
    return out


# ---------------------------------------------------------------------------
# Config C4: keyed join (operators/__init__.py:2075-2190 `_JoinState`, `_JoinLogic`)
# ---------------------------------------------------------------------------


def run_join(batches, insert_mode: str = "last", emit_mode: str = "complete", eof: bool = True):
    """Two-sided join.  ``batches`` = [(keys, sides, vals), ...] in arrival order (the merged, side-labelled
    stream of `_join_label_merge`, operators/__init__.py:2193-2204).  Returns per activation a list of
    ``(key, left_or_None, right_or_None)`` in the engine's order: ascending key string, then item order."""
    assert insert_mode in ("first", "last")
    states: Dict[str, list] = {}
    ids: Dict[str, int] = {}
    acts = []
    for keys, sides, vals in batches:
        grouped: Dict[str, list] = {}
        for k, s, v in zip(keys, sides, vals):
            ks = key_str(k)
            ids[ks] = int(k)
            grouped.setdefault(ks, []).append((int(s), int(v)))
        rows = []
        for ks in sorted(grouped):
            for side, v in grouped[ks]:
                st = states.get(ks)
                if st is None:  # builder(None): fresh _JoinState (also after a DISCARD mid-batch, :1029-1042)
                    st = states[ks] = [None, None]
                if insert_mode == "first":
                    if st[side] is None:
                        st[side] = v
                else:
                    st[side] = v
                if emit_mode == "complete" and st[0] is not None and st[1] is not None:
                    rows.append((ids[ks], st[0], st[1]))
                    del states[ks]
                elif emit_mode == "running":
                    rows.append((ids[ks], st[0], st[1]))
        acts.append(rows)
    if eof:
        rows = []
        if emit_mode == "final":
            for ks in sorted(states):
                st = states[ks]
                rows.append((ids[ks], st[0], st[1]))
            states.clear()
        acts.append(rows)
    return acts
