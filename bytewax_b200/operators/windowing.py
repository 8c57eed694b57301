"""Time-based windowing operators: host-side mirror of ``bytewax.operators.windowing``.

Public names, arguments, sub-step ids (``fold_window`` -> ``window`` ->
``stateful_batch`` / ``unwrap_down`` / ``unwrap_late`` / ``unwrap_meta``,
pysrc/bytewax/operators/windowing.py:1321-1338, 1846) and per-key semantics follow
bytewax v0.21.1.  The generic logic classes below run any Python fold on the
host engine; numeric folds additionally carry a ``GpuFoldPlan`` on their
builder so the engine can hand whole epochs to ``libbwgpu`` (the CUDA path)
instead of calling Python per key.
"""

from __future__ import annotations

import copy
import operator as _pyop
from abc import ABC, abstractmethod
from dataclasses import dataclass, field
from datetime import datetime, timedelta, timezone
from functools import partial
from typing import Any, Callable, Dict, Generic, Iterable, List, Optional, Set, Tuple, TypeVar

import bytewax_b200.operators as op
from bytewax_b200.dataflow import Stream, operator
from bytewax_b200.operators import (
    _EMPTY,
    KeyedStream,
    StatefulBatchLogic,
    _get_system_utc,
    _identity,
    _JoinState,
    _untyped_none,
)

V = TypeVar("V")
W = TypeVar("W")
S = TypeVar("S")

ZERO_TD: timedelta = timedelta(seconds=0)
UTC_MAX: datetime = datetime.max.replace(tzinfo=timezone.utc)
UTC_MIN: datetime = datetime.min.replace(tzinfo=timezone.utc)
LATE_SESSION_ID: int = -1


# ---------------------------------------------------------------------------
# clocks (windowing.py:78-420)
# ---------------------------------------------------------------------------


class ClockLogic(ABC, Generic[V, S]):
    @abstractmethod
    def before_batch(self) -> None: ...

    @abstractmethod
    def on_item(self, value: V) -> Tuple[datetime, datetime]: ...

    @abstractmethod
    def on_notify(self) -> datetime: ...

    @abstractmethod
    def on_eof(self) -> datetime: ...

    @abstractmethod
    def to_system_utc(self, timestamp: datetime) -> Optional[datetime]: ...

    @abstractmethod
    def snapshot(self) -> S: ...


class Clock(ABC, Generic[V, S]):
    @abstractmethod
    def build(self, resume_state: Optional[S]) -> ClockLogic[V, S]: ...


@dataclass
class _SystemClockLogic(ClockLogic):
    """Timestamp == watermark == system time (windowing.py:190-221)."""

    now_getter: Callable[[], datetime]
    _now: datetime = field(init=False)

    def __post_init__(self):
        self._now = self.now_getter()

    def before_batch(self):
        self._now = self.now_getter()

    def on_item(self, value):
        return (self._now, self._now)

    def on_notify(self):
        self._now = self.now_getter()
        return self._now

    def on_eof(self):
        return UTC_MAX

    def to_system_utc(self, timestamp):
        return timestamp

    def snapshot(self):
        return None


@dataclass
class SystemClock(Clock):
    def build(self, resume_state):
        return _SystemClockLogic(_get_system_utc)


@dataclass
class _EventClockState:
    system_time_of_max_event: datetime
    watermark_base: datetime


@dataclass
class _EventClockLogic(ClockLogic):
    """Watermark = max event time - wait + system time elapsed since (windowing.py:230-310)."""

    now_getter: Callable[[], datetime]
    timestamp_getter: Callable[[Any], datetime]
    to_system: Callable[[datetime], Optional[datetime]]
    wait_for_system_duration: timedelta
    state: _EventClockState = field(default_factory=lambda: _EventClockState(UTC_MIN, UTC_MIN))
    _system_now: datetime = field(init=False)

    def __post_init__(self):
        self._system_now = self.now_getter()
        if self.state.system_time_of_max_event <= UTC_MIN:
            self.state.system_time_of_max_event = self._system_now

    def before_batch(self):
        now = self.now_getter()
        if now > self._system_now:  # never let "now" run backwards
            self._system_now = now

    def _watermark(self) -> datetime:
        return self.state.watermark_base + (self._system_now - self.state.system_time_of_max_event)

    def on_item(self, value):
        ts = self.timestamp_getter(value)
        watermark = self._watermark()
        try:
            cand = ts - self.wait_for_system_duration
        except OverflowError:
            cand = None  # unrepresentable: keep advancing from the old base
        if cand is not None and cand > watermark:
            self.state.watermark_base = cand
            self.state.system_time_of_max_event = self._system_now
            return ts, cand
        return ts, watermark

    def on_notify(self):
        self.before_batch()
        return self._watermark()

    def on_eof(self):
        return UTC_MAX

    def to_system_utc(self, timestamp):
        return self.to_system(timestamp)

    def snapshot(self):
        return copy.deepcopy(self.state)


@dataclass
class EventClock(Clock):
    """Use a timestamp embedded in each item (windowing.py:365-420)."""

    ts_getter: Callable[[Any], datetime]
    wait_for_system_duration: timedelta
    now_getter: Callable[[], datetime] = _get_system_utc
    to_system_utc: Callable[[datetime], Optional[datetime]] = _identity

    def build(self, resume_state):
        if resume_state is None:
            return _EventClockLogic(self.now_getter, self.ts_getter, self.to_system_utc, self.wait_for_system_duration)
        return _EventClockLogic(self.now_getter, self.ts_getter, self.to_system_utc, self.wait_for_system_duration, resume_state)


# ---------------------------------------------------------------------------
# windowers (windowing.py:423-950)
# ---------------------------------------------------------------------------


@dataclass
class WindowMetadata:
    open_time: datetime
    close_time: datetime
    merged_ids: Set[int] = field(default_factory=set)


class WindowerLogic(ABC, Generic[S]):
    @abstractmethod
    def open_for(self, timestamp: datetime) -> Iterable[int]: ...

    @abstractmethod
    def late_for(self, timestamp: datetime) -> Iterable[int]: ...

    @abstractmethod
    def merged(self) -> Iterable[Tuple[int, int]]: ...

    @abstractmethod
    def close_for(self, watermark: datetime) -> Iterable[Tuple[int, WindowMetadata]]: ...

    @abstractmethod
    def notify_at(self) -> Optional[datetime]: ...

    @abstractmethod
    def is_empty(self) -> bool: ...

    @abstractmethod
    def snapshot(self) -> S: ...


class Windower(ABC, Generic[S]):
    @abstractmethod
    def build(self, resume_state: Optional[S]) -> WindowerLogic[S]: ...


@dataclass
class _SlidingWindowerState:
    opened: Dict[int, WindowMetadata] = field(default_factory=dict)


@dataclass
class _SlidingWindowerLogic(WindowerLogic):
    """Fixed-size windows every ``offset`` (windowing.py:603-668)."""

    length: timedelta
    offset: timedelta
    align_to: datetime
    state: _SlidingWindowerState

    def intersects(self, timestamp: datetime) -> List[int]:
        since = timestamp - self.align_to
        first = (since - self.length) // self.offset + 1  # timedelta // floors toward -inf
        last = since // self.offset
        return list(range(first, last + 1))

    def _metadata_for(self, window_id: int) -> WindowMetadata:
        open_time = self.align_to + self.offset * window_id
        return WindowMetadata(open_time, open_time + self.length)

    def open_for(self, timestamp):
        ids = self.intersects(timestamp)
        for wid in ids:
            if wid not in self.state.opened:
                self.state.opened[wid] = self._metadata_for(wid)
        return ids

    def late_for(self, timestamp):
        return self.intersects(timestamp)

    def merged(self):
        return _EMPTY

    def close_for(self, watermark):
        done = [(wid, meta) for wid, meta in self.state.opened.items() if meta.close_time <= watermark]
        for wid, _ in done:
            del self.state.opened[wid]
        return done

    def notify_at(self):
        return min((meta.close_time for meta in self.state.opened.values()), default=None)

    def is_empty(self):
        return not self.state.opened

    def snapshot(self):
        return copy.deepcopy(self.state)


@dataclass
class SlidingWindower(Windower):
    length: timedelta
    offset: timedelta
    align_to: datetime

    def __post_init__(self):
        if self.offset > self.length:
            raise ValueError("sliding window `offset` can't be longer than `length`; there would be gaps between windows")

    def build(self, resume_state):
        state = resume_state if resume_state is not None else _SlidingWindowerState()
        return _SlidingWindowerLogic(self.length, self.offset, self.align_to, state)


@dataclass
class TumblingWindower(Windower):
    """Sliding windower with ``offset == length`` (windowing.py:921-926)."""

    length: timedelta
    align_to: datetime

    def build(self, resume_state):
        state = resume_state if resume_state is not None else _SlidingWindowerState()
        return _SlidingWindowerLogic(self.length, self.length, self.align_to, state)


@dataclass
class _SessionWindowerState:
    max_key: int = LATE_SESSION_ID
    sessions: Dict[int, WindowMetadata] = field(default_factory=dict)
    merge_queue: List[Tuple[int, int]] = field(default_factory=list)


def _session_find_merges(sessions: Dict[int, WindowMetadata], gap: timedelta) -> List[Tuple[int, int]]:
    """Merge sessions closer than ``gap``; mutates ``sessions`` (windowing.py:690-720)."""
    merges: List[Tuple[int, int]] = []
    ordered = sorted(sessions.items(), key=lambda kv: kv[1].open_time)
    keep_id, keep = ordered[0]
    for wid, meta in ordered[1:]:
        if meta.open_time - keep.close_time <= gap:
            if meta.close_time > keep.close_time:
                keep.close_time = meta.close_time
            keep.merged_ids.add(wid)
            merges.append((wid, keep_id))
            del sessions[wid]
        else:
            keep_id, keep = wid, meta
    return merges


@dataclass
class _SessionWindowerLogic(WindowerLogic):
    """Activity sessions separated by ``gap`` (windowing.py:723-810).  Host path only."""

    gap: timedelta
    state: _SessionWindowerState

    def _find_merges(self):
        if len(self.state.sessions) >= 2:
            self.state.merge_queue.extend(_session_find_merges(self.state.sessions, self.gap))

    def open_for(self, timestamp):
        for wid, meta in self.state.sessions.items():
            before, after = meta.open_time - timestamp, timestamp - meta.close_time
            if before <= ZERO_TD and after <= ZERO_TD:
                return (wid,)
            if ZERO_TD < before <= self.gap:
                meta.open_time = timestamp
                self._find_merges()
                return (wid,)
            if ZERO_TD < after <= self.gap:
                meta.close_time = timestamp
                self._find_merges()
                return (wid,)
        self.state.max_key += 1
        wid = self.state.max_key
        self.state.sessions[wid] = WindowMetadata(timestamp, timestamp)
        return (wid,)

    def late_for(self, timestamp):
        return (LATE_SESSION_ID,)

    def merged(self):
        out, self.state.merge_queue = self.state.merge_queue, []
        return out

    def close_for(self, watermark):
        try:
            limit = watermark - self.gap
        except OverflowError:
            limit = UTC_MIN
        done = [(wid, meta) for wid, meta in self.state.sessions.items() if meta.close_time < limit]
        for wid, _ in done:
            del self.state.sessions[wid]
        return done

    def notify_at(self):
        first = min((m.close_time for m in self.state.sessions.values()), default=None)
        return first + self.gap if first is not None else None

    def is_empty(self):
        return False  # ids must never be re-used (windowing.py:801-807)

    def snapshot(self):
        return copy.deepcopy(self.state)


@dataclass
class SessionWindower(Windower):
    gap: timedelta

    def __post_init__(self):
        if self.gap < ZERO_TD:
            raise ValueError("session window `gap` must be positive")

    def build(self, resume_state):
        state = resume_state if resume_state is not None else _SessionWindowerState()
        return _SessionWindowerLogic(self.gap, state)


# ---------------------------------------------------------------------------
# the window operator (windowing.py:953-1338)
# ---------------------------------------------------------------------------


class WindowLogic(ABC, Generic[V, W, S]):
    @abstractmethod
    def on_value(self, value: V) -> Iterable[W]: ...

    @abstractmethod
    def on_merge(self, original: "WindowLogic") -> Iterable[W]: ...

    @abstractmethod
    def on_close(self) -> Iterable[W]: ...

    @abstractmethod
    def snapshot(self) -> S: ...


@dataclass(frozen=True)
class _WindowSnapshot:
    clock_state: Any
    windower_state: Any
    logic_states: Dict[int, Any]
    queue: List[Tuple[Any, datetime]]


@dataclass
class _WindowLogic(StatefulBatchLogic):
    """One key's clock + windower + per-window logics (windowing.py:1046-1190)."""

    clock: ClockLogic
    windower: WindowerLogic
    builder: Callable[[Optional[Any]], WindowLogic]
    ordered: bool
    logics: Dict[int, WindowLogic] = field(default_factory=dict)
    queue: List[Tuple[Any, datetime]] = field(default_factory=list)
    _last_watermark: datetime = UTC_MIN

    def _flush(self, watermark: datetime) -> List[Tuple[int, str, Any]]:
        if self.ordered:
            due = [e for e in self.queue if e[1] <= watermark]
            self.queue = [e for e in self.queue if not e[1] <= watermark]
            due.sort(key=lambda e: e[1])
        else:
            due, self.queue = self.queue, []
        events: List[Tuple[int, str, Any]] = []
        for value, ts in due:
            for wid in self.windower.open_for(ts):
                logic = self.logics.get(wid)
                if logic is None:
                    logic = self.logics[wid] = self.builder(None)
                events.extend((wid, "E", w) for w in logic.on_value(value))
        for orig, target in self.windower.merged():
            if target != orig:
                gone = self.logics.pop(orig)
                events.extend((target, "E", w) for w in self.logics[target].on_merge(gone))
        for wid, meta in self.windower.close_for(watermark):
            logic = self.logics.pop(wid)
            events.extend((wid, "E", w) for w in logic.on_close())
            events.append((wid, "M", meta))
        return events

    def _is_empty(self) -> bool:
        return not self.logics and not self.queue and self.windower.is_empty()

    def on_batch(self, values):
        self.clock.before_batch()
        events: List[Tuple[int, str, Any]] = []
        watermark = self._last_watermark
        for value in values:
            ts, watermark = self.clock.on_item(value)
            assert watermark >= self._last_watermark
            self._last_watermark = watermark
            if ts < watermark:
                events.extend((wid, "L", value) for wid in self.windower.late_for(ts))
            else:
                self.queue.append((value, ts))
        events.extend(self._flush(watermark))
        return (events, self._is_empty())

    def on_notify(self):
        watermark = self.clock.on_notify()
        assert watermark >= self._last_watermark
        self._last_watermark = watermark
        return (self._flush(watermark), self._is_empty())

    def on_eof(self):
        watermark = self.clock.on_eof()
        self._last_watermark = watermark
        return (self._flush(watermark), self._is_empty())

    def notify_at(self):
        at = self.windower.notify_at()
        if self.ordered and self.queue:
            q_at = self.queue[0][1]
            at = q_at if at is None else min(at, q_at)
        return self.clock.to_system_utc(at) if at is not None else None

    def snapshot(self):
        return _WindowSnapshot(
            self.clock.snapshot(), self.windower.snapshot(), {wid: lg.snapshot() for wid, lg in self.logics.items()}, list(self.queue)
        )


@dataclass(frozen=True)
class WindowOut(Generic[V, W]):
    """Streams of a windowing operator (windowing.py:1193-1222)."""

    down: KeyedStream
    late: KeyedStream
    meta: KeyedStream


def _unwrap(tag: str, ev):
    if isinstance(ev, WindowColumns):  # columnar egress of `fold_columns` (the CUDA path): a whole stream's rows at once
        return ev if ev.tag == tag else None
    wid, typ, obj = ev
    return (wid, obj) if typ == tag else None


@dataclass
class WindowColumns:
    """One activation's rows of one output stream of `fold_columns(..., columns_out=True)` as numpy columns instead of
    one Python tuple per row.  ``tag``: "E" closed windows (``values`` = accumulators), "L" late items (``values`` = the
    late values), "M" metadata (``open_us`` / ``close_us``).  Item keys are ``str(key)``; ``rows()`` gives the tuples the
    per-item streams would carry, in the same order."""

    tag: str
    keys: Any
    window_ids: Any
    values: Any = None
    open_us: Any = None
    close_us: Any = None

    def __len__(self):
        return len(self.keys)

    def rows(self) -> list:
        ks, ws = [str(int(k)) for k in self.keys], [int(w) for w in self.window_ids]
        if self.tag == "M":
            return [(k, (w, WindowMetadata(_COL_EPOCH + timedelta(microseconds=int(o)), _COL_EPOCH + timedelta(microseconds=int(c)))))
                    for k, w, o, c in zip(ks, ws, self.open_us, self.close_us)]
        return [(k, (w, v)) for k, w, v in zip(ks, ws, self.values.tolist())]


_COL_EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)


@dataclass(frozen=True)
class GpuFoldPlan:
    """What the engine needs to run a windowed numeric fold on ``libbwgpu``.

    Attached to the ``stateful_batch`` builder by the numeric composites below;
    absent for arbitrary Python folds (those stay on the host path).
    """

    reduction: str  # count | sum | min | max
    clock: Any
    windower: Any
    ordered: bool
    value_of: Callable[[Any], Any]  # item value -> number folded
    columns_out: bool = False       # emit WindowColumns items instead of one tuple per row (`fold_columns`)


@operator
def window(step_id: str, up: KeyedStream, clock: Clock, windower: Windower, builder: Callable[[Optional[Any]], WindowLogic],
           ordered: bool = True, _gpu_plan: Optional[GpuFoldPlan] = None, _gpu_session_collect_plan=None) -> WindowOut:
    """Generic windowing operator (windowing.py:1254)."""

    def shim_builder(resume_state):
        if resume_state is None:
            return _WindowLogic(clock.build(None), windower.build(None), builder, ordered)
        logics = {wid: builder(st) for wid, st in resume_state.logic_states.items()}
        return _WindowLogic(
            clock.build(resume_state.clock_state), windower.build(resume_state.windower_state), builder, ordered, logics,
            resume_state.queue,
        )

    shim_builder._gpu_plan = _gpu_plan  # read by bytewax_b200.engine
    shim_builder._gpu_session_collect_plan = _gpu_session_collect_plan  # (engine: read after `_gpu_plan`)
    events = op.stateful_batch("stateful_batch", up, shim_builder)
    downs = op.filter_map_value("unwrap_down", events, partial(_unwrap, "E"))
    lates = op.filter_map_value("unwrap_late", events, partial(_unwrap, "L"))
    metas = op.filter_map_value("unwrap_meta", events, partial(_unwrap, "M"))
    return WindowOut(downs, lates, metas)


@dataclass
class _FoldWindowLogic(WindowLogic):
    """windowing.py:1692-1714."""

    folder: Callable[[Any, Any], Any]
    merger: Callable[[Any, Any], Any]
    state: Any

    def on_value(self, value):
        self.state = self.folder(self.state, value)
        return _EMPTY

    def on_merge(self, consume):
        self.state = self.merger(self.state, consume.state)
        return _EMPTY

    def on_close(self):
        return (self.state,)

    def snapshot(self):
        return copy.deepcopy(self.state)


@operator
def fold_window(step_id: str, up: KeyedStream, clock: Clock, windower: Windower, builder: Callable[[], Any],
                folder: Callable[[Any, Any], Any], merger: Callable[[Any, Any], Any], ordered: bool = True,
                _gpu_plan: Optional[GpuFoldPlan] = None, _gpu_session_collect_plan=None) -> WindowOut:
    """Build an accumulator per window (windowing.py:1717)."""

    def shim_builder(resume_state):
        state = resume_state if resume_state is not None else builder()
        return _FoldWindowLogic(folder, merger, state)

    return window("window", up, clock, windower, shim_builder, ordered, _gpu_plan, _gpu_session_collect_plan)


def _plan_for(reduction: str, clock, windower, ordered, value_of=_identity) -> Optional[GpuFoldPlan]:
    # (SystemClock == an event clock whose timestamps are the arrival times, wait 0: every item is at the watermark)
    # An identity `to_system_utc` only: the device's notify phase compares a window's close, in event time, with the
    # system clock directly, where the reference passes it through `to_system_utc` first (windowing.py:1177-1178).
    identity_utc = isinstance(clock, SystemClock) or (isinstance(clock, EventClock) and clock.to_system_utc is _identity)
    if identity_utc and isinstance(windower, (SlidingWindower, TumblingWindower)):
        return GpuFoldPlan(reduction, clock, windower, ordered, value_of)
    # session windows (K7): unordered only, and likewise an identity `to_system_utc`
    if isinstance(windower, SessionWindower) and not ordered and identity_utc:
        return GpuFoldPlan(reduction, clock, windower, ordered, value_of)
    return None


_COLUMN_FOLDS = {
    # reduction -> (builder, folder over (ts_us, value) items, merger)
    "count": (lambda: 0, lambda a, _v: a + 1, _pyop.add),
    "sum": (lambda: None, lambda a, v: v[1] if a is None else a + v[1], _pyop.add),
    "min": (lambda: None, lambda a, v: v[1] if a is None else min(a, v[1]), min),
    "max": (lambda: None, lambda a, v: v[1] if a is None else max(a, v[1]), max),
}


@operator
def fold_columns(step_id: str, up: Stream, reduction: str, windower: Windower, wait: timedelta = ZERO_TD, ordered: bool = False,
                 columns_out: bool = False, now_getter: Optional[Callable[[], datetime]] = None) -> WindowOut:
    """Windowed ``count`` / ``sum`` / ``min`` / ``max`` by key over a stream of `bytewax_b200.inputs.KeyedColumns` items (this
    package's columnar ingest contract, SURVEY 8f row 1): every item is a whole batch -- ``keys`` (uint64; the item key is
    ``str(key)``), ``ts_us`` (event time), ``vals`` -- and becomes ONE activation of the CUDA fold, with no Python object per row.
    Same semantics as ``count_window`` / ``reduce_window`` over the rows ``(str(key), value)`` with an `EventClock` on ``ts_us``:
    without the CUDA path the engine expands the columns into exactly those items and runs the host logic.

    ``columns_out=True``: on the CUDA path the three output streams carry one `WindowColumns` item per activation (numpy columns;
    ``.rows()`` gives the tuples) instead of one tuple per row."""
    if reduction not in _COLUMN_FOLDS:
        raise ValueError(f"unknown reduction {reduction!r}; one of {sorted(_COLUMN_FOLDS)}")
    if not isinstance(windower, (SlidingWindower, TumblingWindower)):
        raise TypeError("fold_columns needs a SlidingWindower or TumblingWindower")
    kw = {} if now_getter is None else {"now_getter": now_getter}
    clock = EventClock(lambda v: _COL_EPOCH + timedelta(microseconds=int(v[0])), wait, **kw)
    builder, folder, merger = _COLUMN_FOLDS[reduction]
    keyed = op.key_on("batch", up, lambda _cols: "cols")  # (key, KeyedColumns): the stateful step takes it from here
    plan = GpuFoldPlan(reduction, clock, windower, ordered, lambda v: v[1], columns_out)
    return fold_window("fold", keyed, clock, windower, builder, folder, merger, ordered=ordered, _gpu_plan=plan)


@operator
def count_window(step_id: str, up: Stream, clock: Clock, windower: Windower, key: Callable[[Any], str]) -> WindowOut:
    """Count items per key per window (windowing.py:1579)."""
    keyed = op.key_on("keyed", up, key)
    return fold_window(
        "sum", keyed, clock, windower, lambda: 0, lambda s, _: s + 1, lambda s, t: s + t, ordered=False,
        _gpu_plan=_plan_for("count", clock, windower, False),
    )


_NUMERIC_REDUCERS = {_pyop.add: "sum", max: "max", min: "min"}


@operator
def reduce_window(step_id: str, up: KeyedStream, clock: Clock, windower: Windower, reducer: Callable[[Any, Any], Any],
                  _gpu_plan: Optional[GpuFoldPlan] = None) -> WindowOut:
    """Combine values per window; the first value seeds it (windowing.py:2239)."""

    def shim_folder(s, v):
        return v if s is None else reducer(s, v)

    plan = _gpu_plan
    if plan is None and reducer in _NUMERIC_REDUCERS:
        plan = _plan_for(_NUMERIC_REDUCERS[reducer], clock, windower, False)
    return fold_window("fold_window", up, clock, windower, _untyped_none, shim_folder, reducer, ordered=False, _gpu_plan=plan)


@dataclass(frozen=True)
class GpuArgWindowPlan:
    """A ``max_window`` / ``min_window`` with a ``by=`` projection the engine may run with ``bw_argwin_*`` (K11): a
    tumbling, sliding or session windower and an `EventClock` with an identity ``to_system_utc`` or a `SystemClock`.
    Items travel as handles into a host-side dict with the number ``by`` gives each; ``by`` runs once per item at
    ingest, so it must be pure and defined on every item, late ones included."""

    extreme: str  # max | min
    by: Callable[[Any], Any]
    clock: Any
    windower: Any


def _arg_window_plan(extreme, by, clock, windower) -> Optional[GpuArgWindowPlan]:
    # a custom `to_system_utc` moves the notify time away from the event time the device compares with the system clock
    # (windowing.py:1177-1178): host engine
    if not isinstance(windower, (SlidingWindower, TumblingWindower, SessionWindower)):
        return None
    if not (isinstance(clock, SystemClock) or (isinstance(clock, EventClock) and clock.to_system_utc is _identity)):
        return None
    return GpuArgWindowPlan(extreme, by, clock, windower)


@operator
def max_window(step_id: str, up: KeyedStream, clock: Clock, windower: Windower, by: Callable[[Any], Any] = _identity) -> WindowOut:
    """windowing.py:2145."""
    plan = _plan_for("max", clock, windower, False) if by is _identity else _arg_window_plan("max", by, clock, windower)
    return reduce_window("reduce_window", up, clock, windower, partial(max, key=by), _gpu_plan=plan)


@operator
def min_window(step_id: str, up: KeyedStream, clock: Clock, windower: Windower, by: Callable[[Any], Any] = _identity) -> WindowOut:
    """windowing.py:2192."""
    plan = _plan_for("min", clock, windower, False) if by is _identity else _arg_window_plan("min", by, clock, windower)
    return reduce_window("reduce_window", up, clock, windower, partial(min, key=by), _gpu_plan=plan)


def _collect_list_folder(s: list, v):
    s.append(v)
    return s


def _collect_set_folder(s: set, v):
    s.add(v)
    return s


def _collect_dict_folder(d: dict, k_v):
    k, v = k_v
    d[k] = v
    return d


def _collect_dict_merger(a: dict, b: dict):
    a.update(b)
    return a


@operator
def collect_window(step_id: str, up: KeyedStream, clock: Clock, windower: Windower, into=list, ordered: bool = True) -> WindowOut:
    """Collect a window's items into a list / set / dict (windowing.py:1436)."""
    if issubclass(into, list):
        folder, merger = _collect_list_folder, (lambda a, b: a + b)
    elif issubclass(into, set):
        folder, merger = _collect_set_folder, (lambda a, b: a | b)
    elif issubclass(into, dict):
        folder, merger = _collect_dict_folder, _collect_dict_merger
    else:
        raise TypeError(f"`collect_window` doesn't support `{into:!}`; only `set`, `list`, and `dict`; use `fold_window` directly")
    return fold_window("fold_window", up, clock, windower, into, folder, merger, ordered,
                       _gpu_plan=_collect_window_plan(step_id, clock, windower, into, ordered),
                       _gpu_session_collect_plan=_session_collect_window_plan(step_id, clock, windower, into, ordered))


@dataclass(frozen=True)
class GpuCollectWindowPlan:
    """A ``collect_window`` the engine may run with ``bw_collect_*`` (K9): ``into`` exactly `list`, `set` or `dict`, a
    tumbling or sliding windower, and an `EventClock` with an identity ``to_system_utc`` or a `SystemClock`.  Values travel
    as handles into a host-side dict; each window's container is built from its handles in play order."""

    into: type
    ordered: bool
    clock: Any
    windower: Any
    step_id: str = ""  # the `collect_window` step id, for the reference's `dict` error message


def _collect_window_plan(step_id, clock, windower, into, ordered) -> Optional[GpuCollectWindowPlan]:
    # the reference builds the plain type even for a subclass `into` (windowing.py:1356-1384) while this mirror builds
    # `into` itself: a subclass stays on the host engine.  Session windows merge, and a custom `to_system_utc` moves the
    # notify time away from the event time the device compares with the system clock (windowing.py:1177-1178).
    if into not in (list, set, dict):
        return None
    if not isinstance(windower, (SlidingWindower, TumblingWindower)):
        return None
    if not (isinstance(clock, SystemClock) or (isinstance(clock, EventClock) and clock.to_system_utc is _identity)):
        return None
    return GpuCollectWindowPlan(into, bool(ordered), clock, windower, step_id)


@dataclass(frozen=True)
class GpuSessionCollectWindowPlan:
    """A ``collect_window`` over a `SessionWindower` the engine may run with ``bw_scwin_*`` (K12): ``into`` exactly
    `list`, `set` or `dict`, and an `EventClock` with an identity ``to_system_utc`` or a `SystemClock`.  Values travel as
    handles into a host-side dict; each session's container is built from its handles in flattened play order, with the
    merger applied where each merged-away session's block sits.  It rides on the builder's own attribute,
    ``_gpu_session_collect_plan``, beside ``_gpu_plan`` (which session collects never carry)."""

    into: type
    ordered: bool
    clock: Any
    windower: Any
    step_id: str = ""  # the `collect_window` step id, for the reference's `dict` error message


def _session_collect_window_plan(step_id, clock, windower, into, ordered) -> Optional[GpuSessionCollectWindowPlan]:
    # the conditions of `_collect_window_plan`, over a session windower
    if into not in (list, set, dict) or not isinstance(windower, SessionWindower):
        return None
    if not (isinstance(clock, SystemClock) or (isinstance(clock, EventClock) and clock.to_system_utc is _identity)):
        return None
    return GpuSessionCollectWindowPlan(into, bool(ordered), clock, windower, step_id)


@dataclass
class _JoinWindowLogic(WindowLogic):
    """windowing.py:1849-1902."""

    insert_mode: str
    emit_mode: str
    state: _JoinState

    def on_value(self, value):
        side, v = value
        if self.insert_mode == "first" and not self.state.is_set(side):
            self.state.set_val(side, v)
        elif self.insert_mode == "last":
            self.state.set_val(side, v)
        elif self.insert_mode == "product":
            self.state.add_val(side, v)
        if self.emit_mode == "complete" and self.state.all_set():
            rows = self.state.astuples()
            self.state.clear()
            return rows
        if self.emit_mode == "running":
            return self.state.astuples()
        return _EMPTY

    def on_merge(self, original):
        # windowing.py:1879-1891: "first" takes the merged-away session's value on every side it set; "last" keeps the
        # survivor's value on every side the survivor set
        if self.insert_mode == "first":
            self.state |= original.state
        elif self.insert_mode == "last":
            original.state |= self.state
            self.state = original.state
        else:
            self.state += original.state
        if self.emit_mode == "complete" and self.state.all_set():
            rows = self.state.astuples()
            self.state.clear()
            return rows
        if self.emit_mode == "running":
            return self.state.astuples()
        return _EMPTY

    def on_close(self):
        return self.state.astuples() if self.emit_mode == "final" else _EMPTY

    def snapshot(self):
        return copy.deepcopy(self.state)


@operator
def join_window(step_id: str, clock: Clock, windower: Windower, *sides: KeyedStream, insert_mode: str = "last",
                emit_mode: str = "final", ordered: bool = True) -> WindowOut:
    """Join keyed streams within windows (windowing.py:2055).  The clock sees the bare value."""
    if insert_mode not in ("first", "last", "product"):
        raise ValueError(f"unknown join insert mode {insert_mode!r}")
    if emit_mode not in ("complete", "final", "running"):
        raise ValueError(f"unknown join emit mode {emit_mode!r}")
    side_count = len(sides)

    def shim_builder(resume_state):
        state = resume_state if resume_state is not None else _JoinState.for_side_count(side_count)
        return _JoinWindowLogic(insert_mode, emit_mode, state)

    plan = (_join_window_plan(clock, windower, side_count, insert_mode, emit_mode, ordered)
            or _session_product_join_window_plan(clock, windower, side_count, insert_mode, emit_mode, ordered))
    # items reach the clock as (side, value): unwrap for the user's ts_getter
    if isinstance(clock, EventClock):
        inner = clock.ts_getter
        clock = EventClock(lambda side_v: inner(side_v[1]), clock.wait_for_system_duration, clock.now_getter, clock.to_system_utc)
    merged = op._join_label_merge("add_names", *sides)
    return window("window", merged, clock, windower, shim_builder, ordered=ordered, _gpu_plan=plan)


@dataclass(frozen=True)
class GpuJoinWindowPlan:
    """A ``join_window`` the engine may run on the device: insert mode first / last with ``bw_jwin_*`` (K8, tumbling or
    sliding windower) or ``bw_sjwin_*`` (K10, `SessionWindower`), insert mode product with ``bw_pjwin_*`` (K14, tumbling or
    sliding windower) or ``bw_spjwin_*`` (K16, `SessionWindower`); 1 to 4 sides, and an `EventClock` with an identity
    ``to_system_utc`` or a `SystemClock`.  Values travel as handles into a host-side dict, so they can be any Python
    object."""

    insert_mode: str
    emit_mode: str
    ordered: bool
    sides: int
    clock: Any     # the user's clock: its ts_getter sees the bare value
    windower: Any


def _join_window_plan(clock, windower, side_count, insert_mode, emit_mode, ordered) -> Optional[GpuJoinWindowPlan]:
    # the plans of K8, K10 and K14; product over sessions, where a merge concatenates the side lists
    # (`self.state += original.state`), is K16's: `_session_product_join_window_plan`.
    # A custom `to_system_utc` moves the notify time away from the event time the device compares with the system clock
    # (windowing.py:1177-1178): host engine.
    if insert_mode not in ("first", "last", "product") or not 1 <= side_count <= 4:
        return None
    windowers = (SlidingWindower, TumblingWindower) if insert_mode == "product" else (SlidingWindower, TumblingWindower, SessionWindower)
    if not isinstance(windower, windowers):
        return None
    if not (isinstance(clock, SystemClock) or (isinstance(clock, EventClock) and clock.to_system_utc is _identity)):
        return None
    return GpuJoinWindowPlan(insert_mode, emit_mode, bool(ordered), side_count, clock, windower)


def _session_product_join_window_plan(clock, windower, side_count, insert_mode, emit_mode, ordered) -> Optional[GpuJoinWindowPlan]:
    # product over a `SessionWindower` (K16): 1 to 4 sides; a custom `to_system_utc` stays on the host engine, as above
    if insert_mode != "product" or not 1 <= side_count <= 4 or not isinstance(windower, SessionWindower):
        return None
    if not (isinstance(clock, SystemClock) or (isinstance(clock, EventClock) and clock.to_system_utc is _identity)):
        return None
    return GpuJoinWindowPlan(insert_mode, emit_mode, bool(ordered), side_count, clock, windower)
