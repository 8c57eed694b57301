"""Operator library: host-side mirror of ``bytewax.operators``.

Same public names, arguments, step ids (sub-step names are part of the
contract: they appear in ``inspect`` output and recovery keys -- SURVEY.md
Appendix B) and runtime behaviour as pysrc/bytewax/operators/__init__.py of
bytewax v0.21.1, re-authored for this engine.  Eight operators are *core*
(``_core=True``): the engine (bytewax_b200/engine.py) executes those; all the
others only compose them.  Reference line numbers are given per operator.
"""

from __future__ import annotations

import copy
import itertools
import operator as _pyop
from abc import ABC, abstractmethod
from dataclasses import dataclass, field
from datetime import datetime, timedelta, timezone
from functools import partial
from typing import Any, Callable, Dict, Generic, Iterable, List, Optional, Tuple, TypeVar

from bytewax_b200.dataflow import Dataflow, Stream, f_repr, operator

X = TypeVar("X")
Y = TypeVar("Y")
V = TypeVar("V")
W = TypeVar("W")
S = TypeVar("S")
KeyedStream = Stream  # Stream[Tuple[str, V]]

_EMPTY: Tuple = tuple()


def _identity(x):
    return x


def _untyped_none():
    return None


def _get_system_utc() -> datetime:
    return datetime.now(tz=timezone.utc)


# ---------------------------------------------------------------------------
# core operators (executed by the engine; src/worker.rs:298-466)
# ---------------------------------------------------------------------------


@dataclass(frozen=True)
class BranchOut(Generic[X, Y]):
    """Streams returned by :func:`branch`."""

    trues: Stream
    falses: Stream


@operator(_core=True)
def branch(step_id: str, up: Stream, predicate: Callable[[Any], bool]) -> BranchOut:
    """Split a stream by a predicate (operators/__init__.py:119; src/operators.rs:45-100)."""
    return BranchOut(trues=Stream(f"{step_id}.trues", up._scope), falses=Stream(f"{step_id}.falses", up._scope))


@operator(_core=True)
def flat_map_batch(step_id: str, up: Stream, mapper: Callable[[List[Any]], Iterable[Any]]) -> Stream:
    """One ``mapper(list_of_items)`` call per batch (operators/__init__.py:179; src/operators.rs:135-228)."""
    return Stream(f"{step_id}.down", up._scope)


@operator(_core=True)
def input(step_id: str, flow: Dataflow, source) -> Stream:  # noqa: A001
    """Introduce items from a source (operators/__init__.py:240; src/inputs.rs)."""
    return Stream(f"{step_id}.down", flow._scope)


def _default_debug_inspector(step_id: str, item: Any, epoch: int, worker: int) -> None:
    """What ``inspect_debug`` prints when no inspector is given (operators/__init__.py:292-293)."""
    print(f"{step_id} W{worker} @{epoch}: {item!r}", flush=True)


@operator(_core=True)
def inspect_debug(step_id: str, up: Stream, inspector: Callable[[str, Any, int, int], None] = _default_debug_inspector) -> Stream:
    """``inspector(step_id, item, epoch, worker)`` per item (operators/__init__.py:296; src/operators.rs:242-317)."""
    return Stream(f"{step_id}.down", up._scope)


@operator(_core=True)
def merge(step_id: str, *ups: Stream) -> Stream:
    """Concatenate streams (operators/__init__.py:394; src/operators.rs:331-343)."""
    scopes = {id(u._scope): u._scope for u in ups}
    if len(scopes) != 1:
        raise AssertionError("merged streams must be in the same scope")
    return Stream(f"{step_id}.down", next(iter(scopes.values())))


@operator(_core=True)
def output(step_id: str, up: Stream, sink) -> None:
    """Write items to a sink (operators/__init__.py:449; src/outputs.rs)."""
    return None


@operator(_core=True)
def redistribute(step_id: str, up: Stream) -> Stream:
    """Random exchange across workers (operators/__init__.py:497; src/operators.rs:353-361)."""
    return Stream(f"{step_id}.down", up._scope)


class StatefulBatchLogic(ABC, Generic[V, W, S]):
    """Per-key logic of :func:`stateful_batch` (operators/__init__.py:593-792)."""

    RETAIN: bool = False
    DISCARD: bool = True

    @abstractmethod
    def on_batch(self, values: List[V]) -> Tuple[Iterable[W], bool]: ...

    def on_notify(self) -> Tuple[Iterable[W], bool]:
        return (_EMPTY, StatefulBatchLogic.RETAIN)

    def on_eof(self) -> Tuple[Iterable[W], bool]:
        return (_EMPTY, StatefulBatchLogic.RETAIN)

    def notify_at(self) -> Optional[datetime]:
        return None

    @abstractmethod
    def snapshot(self) -> S: ...


@operator(_core=True)
def stateful_batch(step_id: str, up: KeyedStream, builder: Callable[[Optional[Any]], StatefulBatchLogic]) -> KeyedStream:
    """Keyed stateful step (operators/__init__.py:795; src/operators.rs:549-1038)."""
    return Stream(f"{step_id}.down", up._scope)


# ---------------------------------------------------------------------------
# stateless composites
# ---------------------------------------------------------------------------


@operator
def flat_map(step_id: str, up: Stream, mapper: Callable[[Any], Iterable[Any]]) -> Stream:
    """operators/__init__.py:1615."""

    def shim_mapper(xs):
        return itertools.chain.from_iterable(mapper(x) for x in xs)

    return flat_map_batch("flat_map_batch", up, shim_mapper)


@operator
def flat_map_value(step_id: str, up: KeyedStream, mapper: Callable[[Any], Iterable[Any]]) -> KeyedStream:
    """operators/__init__.py:1676."""

    def shim_mapper(k_v):
        try:
            k, v = k_v
        except TypeError as ex:
            raise TypeError(
                f"step {step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(k_v)!r} instead"
            ) from ex
        return ((k, w) for w in mapper(v))

    return flat_map("flat_map", up, shim_mapper)


@operator
def flatten(step_id: str, up: Stream) -> Stream:
    """operators/__init__.py:1734."""

    def shim_mapper(x):
        if not isinstance(x, Iterable):
            raise TypeError(f"step {step_id!r} requires upstream to be iterables; got a {type(x)!r} instead")
        return x

    return flat_map("flat_map", up, shim_mapper)


@operator
def filter(step_id: str, up: Stream, predicate: Callable[[Any], bool]) -> Stream:  # noqa: A001
    """operators/__init__.py:1776."""

    def shim_mapper(x):
        keep = predicate(x)
        if not isinstance(keep, bool):
            raise TypeError(f"return value of `predicate` {f_repr(predicate)} in step {step_id!r} must be a `bool`; got a {type(keep)!r} instead")
        return (x,) if keep else _EMPTY

    return flat_map("flat_map", up, shim_mapper)


@operator
def filter_value(step_id: str, up: KeyedStream, predicate: Callable[[Any], bool]) -> KeyedStream:
    """operators/__init__.py:1829."""

    def shim_mapper(v):
        keep = predicate(v)
        if not isinstance(keep, bool):
            raise TypeError(f"return value of `predicate` {f_repr(predicate)} in step {step_id!r} must be a `bool`; got a {type(keep)!r} instead")
        return (v,) if keep else _EMPTY

    return flat_map_value("filter", up, shim_mapper)


@operator
def filter_map(step_id: str, up: Stream, mapper: Callable[[Any], Optional[Any]]) -> Stream:
    """operators/__init__.py:1870."""

    def shim_mapper(x):
        y = mapper(x)
        return (y,) if y is not None else _EMPTY

    return flat_map("flat_map", up, shim_mapper)


@operator
def filter_map_value(step_id: str, up: KeyedStream, mapper: Callable[[Any], Optional[Any]]) -> KeyedStream:
    """operators/__init__.py:1904."""

    def shim_mapper(v):
        w = mapper(v)
        return (w,) if w is not None else _EMPTY

    return flat_map_value("flat_map_value", up, shim_mapper)


@operator
def inspect(step_id: str, up: Stream, inspector: Callable[[str, Any], None] = None) -> Stream:
    """operators/__init__.py:2017: default prints ``f"{step_id}: {item!r}"``."""
    if inspector is None:

        def inspector(step, item):
            print(f"{step}: {item!r}", flush=True)

    def shim_inspector(_fq_step_id, item, _epoch, _worker):
        inspector(step_id, item)  # this step's own id, not the inner inspect_debug's (operators/__init__.py:2064-2067)

    return inspect_debug("inspect_debug", up, shim_inspector)


@operator
def key_on(step_id: str, up: Stream, key: Callable[[Any], str]) -> KeyedStream:
    """operators/__init__.py:2401."""

    def shim_mapper(x):
        k = key(x)
        if not isinstance(k, str):
            raise TypeError(f"return value of `key` {f_repr(key)} in step {step_id!r} must be a `str`; got a {type(k)!r} instead")
        return (k, x)

    return map("map", up, shim_mapper)


@operator
def key_rm(step_id: str, up: KeyedStream) -> Stream:
    """operators/__init__.py:2439."""

    def shim_mapper(k_v):
        _k, v = k_v
        return v

    return map("map", up, shim_mapper)


@operator
def map(step_id: str, up: Stream, mapper: Callable[[Any], Any]) -> Stream:  # noqa: A001
    """operators/__init__.py:2479."""

    def shim_mapper(xs):
        return [mapper(x) for x in xs]

    return flat_map_batch("flat_map_batch", up, shim_mapper)


@operator
def map_value(step_id: str, up: KeyedStream, mapper: Callable[[Any], Any]) -> KeyedStream:
    """operators/__init__.py:2557."""

    def shim_mapper(k_v):
        try:
            k, v = k_v
        except TypeError as ex:
            raise TypeError(
                f"step {step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(k_v)!r} instead"
            ) from ex
        return (k, mapper(v))

    return map("map", up, shim_mapper)


class _RaiseSink:
    def __init__(self, step_id: str):
        self.step_id = step_id


@operator
def raises(step_id: str, up: Stream) -> None:
    """Raise on any item (operators/__init__.py:2745)."""
    from bytewax_b200.outputs import DynamicSink, StatelessSinkPartition

    class _Part(StatelessSinkPartition):
        def write_batch(self, items):
            for item in items:
                raise RuntimeError(f"`raises` step {step_id!r} got an item: {item!r}")

    class _Sink(DynamicSink):
        def build(self, _step_id, _worker_index, _worker_count):
            return _Part()

    return output("output", up, _Sink())


class TTLCache(Generic[X, Y]):
    """Time-limited memo of a getter (operators/__init__.py:1275-1344)."""

    def __init__(self, v_getter: Callable[[Any], Any], now_getter: Callable[[], datetime], ttl: timedelta):
        self.v_getter, self.now_getter, self.ttl = v_getter, now_getter, ttl
        self._cache: Dict[Any, Tuple[datetime, Any]] = {}

    def get(self, k):
        now = self.now_getter()
        try:
            ts, v = self._cache[k]
            if now - ts > self.ttl:
                raise KeyError()
        except KeyError:
            v = self.v_getter(k)
            self._cache[k] = (now, v)
        return v

    def remove(self, k):
        del self._cache[k]


@operator
def enrich_cached(step_id: str, up: Stream, getter: Callable[[Any], Any], mapper: Callable[[TTLCache, Any], Any],
                  ttl: timedelta = timedelta.max, _now_getter: Callable[[], datetime] = _get_system_utc) -> Stream:
    """operators/__init__.py:1347."""

    def shim_mapper(xs, cache=None):
        if cache is None:
            cache = shim_mapper._cache  # one cache per step (per worker in the reference)
        return [mapper(cache, x) for x in xs]

    shim_mapper._cache = TTLCache(getter, _now_getter, ttl)
    return flat_map_batch("flat_map_batch", up, shim_mapper)


# ---------------------------------------------------------------------------
# stateful composites
# ---------------------------------------------------------------------------


class StatefulLogic(ABC, Generic[V, W, S]):
    """Per-item logic of :func:`stateful` (operators/__init__.py:918-1021)."""

    RETAIN: bool = False
    DISCARD: bool = True

    @abstractmethod
    def on_item(self, value: V) -> Tuple[Iterable[W], bool]: ...

    def on_notify(self) -> Tuple[Iterable[W], bool]:
        return (_EMPTY, StatefulLogic.RETAIN)

    def on_eof(self) -> Tuple[Iterable[W], bool]:
        return (_EMPTY, StatefulLogic.RETAIN)

    def notify_at(self) -> Optional[datetime]:
        return None

    @abstractmethod
    def snapshot(self) -> S: ...


@dataclass
class _StatefulLogicShim(StatefulBatchLogic):
    """Adapts a per-item logic to the batch protocol (operators/__init__.py:1024-1062)."""

    step_id: str
    builder: Callable[[Optional[Any]], StatefulLogic]
    logic: Optional[StatefulLogic]

    def on_batch(self, values):
        out: List[Any] = []
        for v in values:
            if self.logic is None:  # discarded mid-batch: a fresh one for the next value
                self.logic = self.builder(None)
            ws, discard = self.logic.on_item(v)
            out.extend(ws)
            if discard:
                self.logic = None
        return (out, self.logic is None)

    def on_notify(self):
        assert self.logic is not None
        ws, discard = self.logic.on_notify()
        return (ws, discard)

    def on_eof(self):
        assert self.logic is not None
        ws, discard = self.logic.on_eof()
        return (ws, discard)

    def notify_at(self):
        assert self.logic is not None
        return self.logic.notify_at()

    def snapshot(self):
        assert self.logic is not None
        return self.logic.snapshot()


@dataclass(frozen=True)
class GpuFinalPlan:
    """What the engine needs to run a numeric ``*_final`` fold on ``libbwgpu`` (``bw_fold_spec.ts_source ==
    BW_TS_NONE``): attached to the ``stateful_batch`` builder by ``count_final`` / ``reduce_final(add|max|min)`` /
    ``max_final`` / ``min_final``; absent for arbitrary Python folders, which stay on the host path."""

    reduction: str  # sum | min | max


@operator
def stateful(step_id: str, up: KeyedStream, builder: Callable[[Optional[Any]], StatefulLogic],
             _gpu_plan: Optional[GpuFinalPlan] = None) -> KeyedStream:
    """operators/__init__.py:1065."""

    def shim_builder(resume_state):
        return _StatefulLogicShim(step_id, builder, builder(resume_state))

    shim_builder._gpu_plan = _gpu_plan  # read by bytewax_b200.engine
    return stateful_batch("stateful_batch", up, shim_builder)


@dataclass
class _CollectState(Generic[V]):
    acc: List[V] = field(default_factory=list)
    timeout_at: Optional[datetime] = None


@dataclass
class _CollectLogic(StatefulLogic):
    """operators/__init__.py:1113-1164."""

    step_id: str
    now_getter: Callable[[], datetime]
    timeout: timedelta
    max_size: int
    state: _CollectState

    def on_item(self, value):
        self.state.timeout_at = self.now_getter() + self.timeout
        self.state.acc.append(value)
        if len(self.state.acc) >= self.max_size:
            return ((self.state.acc,), StatefulLogic.DISCARD)
        return (_EMPTY, StatefulLogic.RETAIN)

    def on_notify(self):
        return ((self.state.acc,), StatefulLogic.DISCARD)

    def on_eof(self):
        return ((self.state.acc,), StatefulLogic.DISCARD)

    def notify_at(self):
        return self.state.timeout_at

    def snapshot(self):
        return copy.deepcopy(self.state)


@dataclass(frozen=True)
class GpuCollectPlan:
    """A ``collect`` whose ``max_size`` is an ``int``: the engine may run it with ``bw_kcollect_*`` (K13).  ``max_size`` is
    stored as ``max(1, min(max_size, 2**64 - 1))``, which splits lists exactly where the reference does; values travel as
    handles, so they can be any Python object."""

    timeout: timedelta
    max_size: int


@operator
def collect(step_id: str, up: KeyedStream, timeout: timedelta, max_size: int) -> KeyedStream:
    """operators/__init__.py:1167."""

    def shim_builder(resume_state):
        state = resume_state if resume_state is not None else _CollectState()
        return _CollectLogic(step_id, _get_system_utc, timeout, max_size, state)

    plan = GpuCollectPlan(timeout, max(1, min(max_size, 2**64 - 1))) if isinstance(max_size, int) else None
    return stateful("stateful", up, shim_builder, _gpu_plan=plan)


@operator
def count_final(step_id: str, up: Stream, key: Callable[[Any], str]) -> KeyedStream:
    """operators/__init__.py:1221: ``init_count`` then ``sum``."""
    down = map("init_count", up, lambda x: (key(x), 1))
    return reduce_final("sum", down, lambda s, x: s + x, _gpu_plan=GpuFinalPlan("sum"))


@dataclass
class _FoldFinalLogic(StatefulLogic):
    """operators/__init__.py:1923-1950."""

    step_id: str
    folder: Callable[[Any, Any], Any]
    state: Any

    def on_item(self, value):
        self.state = self.folder(self.state, value)
        return (_EMPTY, StatefulLogic.RETAIN)

    def on_eof(self):
        return ((self.state,), StatefulLogic.DISCARD)

    def snapshot(self):
        return copy.deepcopy(self.state)


@operator
def fold_final(step_id: str, up: KeyedStream, builder: Callable[[], Any], folder: Callable[[Any, Any], Any],
               _gpu_plan: Optional[GpuFinalPlan] = None) -> KeyedStream:
    """operators/__init__.py:1953."""

    def shim_builder(resume_state):
        state = resume_state if resume_state is not None else builder()
        return _FoldFinalLogic(step_id, folder, state)

    return stateful("stateful", up, shim_builder, _gpu_plan)


_NUMERIC_FINAL_REDUCERS = {_pyop.add: "sum", max: "max", min: "min"}


@operator
def reduce_final(step_id: str, up: KeyedStream, reducer: Callable[[Any, Any], Any],
                 _gpu_plan: Optional[GpuFinalPlan] = None) -> KeyedStream:
    """operators/__init__.py:2783: per-batch ``pre_reduce`` combiner, then ``fold_final``."""
    plan = _gpu_plan
    if plan is None and reducer in _NUMERIC_FINAL_REDUCERS:
        plan = GpuFinalPlan(_NUMERIC_FINAL_REDUCERS[reducer])

    def pre_reducer(mixed_batch):
        states: Dict[str, Any] = {}
        for k, v in mixed_batch:
            states[k] = reducer(states[k], v) if k in states else v
        return states.items()

    pre_up = flat_map_batch("pre_reduce", up, pre_reducer)

    def shim_folder(s, v):
        return v if s is None else reducer(s, v)

    return fold_final("fold_final", pre_up, _untyped_none, shim_folder, _gpu_plan=plan)


@operator
def max_final(step_id: str, up: KeyedStream, by: Callable[[Any], Any] = _identity) -> KeyedStream:
    """operators/__init__.py:2624."""
    return reduce_final("reduce_final", up, partial(max, key=by), _gpu_plan=GpuFinalPlan("max") if by is _identity else None)


@operator
def min_final(step_id: str, up: KeyedStream, by: Callable[[Any], Any] = _identity) -> KeyedStream:
    """operators/__init__.py:2685."""
    return reduce_final("reduce_final", up, partial(min, key=by), _gpu_plan=GpuFinalPlan("min") if by is _identity else None)


@dataclass
class _StatefulFlatMapLogic(StatefulLogic):
    """operators/__init__.py:2860-2890."""

    step_id: str
    mapper: Callable[[Optional[Any], Any], Tuple[Optional[Any], Iterable[Any]]]
    state: Optional[Any] = None

    def on_item(self, value):
        res = self.mapper(self.state, value)
        try:
            s, ws = res
        except TypeError as ex:
            raise TypeError(
                f"return value of `mapper` {f_repr(self.mapper)} in step {self.step_id!r} must be a 2-tuple of "
                f"`(updated_state, emit_values)`; got a {type(res)!r} instead"
            ) from ex
        if s is None:
            return (ws, StatefulLogic.DISCARD)
        self.state = s
        return (ws, StatefulLogic.RETAIN)

    def snapshot(self):
        return copy.deepcopy(self.state)


@operator
def stateful_flat_map(step_id: str, up: KeyedStream, mapper: Callable[[Optional[Any], Any], Tuple[Optional[Any], Iterable[Any]]],
                      _gpu_plan: Optional["GpuSmapPlan"] = None) -> KeyedStream:
    """operators/__init__.py:2893."""

    def shim_builder(resume_state):
        return _StatefulFlatMapLogic(step_id, mapper, resume_state)

    return stateful("stateful", up, shim_builder, _gpu_plan)


@dataclass(frozen=True)
class GpuSmapPlan:
    """A ``stateful_map`` whose mapper is a DECLARED detector (``bytewax_b200.detectors.ZScoreDetector``): the engine may
    run the step with ``bw_smap_*`` (K5) instead of calling the mapper item by item.  Arbitrary mappers have no plan."""

    window: int
    threshold: float


@dataclass(frozen=True)
class GpuJoinPlan:
    """A two-sided ``join`` with insert mode first / last: the engine may run it with ``bw_join_*`` (K6); values travel as
    handles into a host-side list, so they can be any Python object."""

    insert_mode: str
    emit_mode: str


@dataclass(frozen=True)
class GpuKeyJoinPlan:
    """A ``join`` with 1 to 4 sides that `GpuJoinPlan` does not cover -- product inserts, and first / last with 1, 3 or 4
    sides: the engine may run it with ``bw_kjoin_*`` (K15); values travel as handles into a host-side dict, so they can
    be any Python object."""

    insert_mode: str
    emit_mode: str
    sides: int


@operator
def stateful_map(step_id: str, up: KeyedStream, mapper: Callable[[Optional[Any], Any], Tuple[Optional[Any], Any]]) -> KeyedStream:
    """operators/__init__.py:2920."""

    def shim_mapper(state, v):
        res = mapper(state, v)
        try:
            s, w = res
        except TypeError as ex:
            raise TypeError(
                f"return value of `mapper` {f_repr(mapper)} in step {step_id!r} must be a 2-tuple of "
                f"`(updated_state, emit_value)`; got a {type(res)!r} instead"
            ) from ex
        return (s, (w,))

    # a declared detector carries its plan (the recogniser of bytewax_b200.engine reads it off the step's builder)
    return stateful_flat_map("stateful_flat_map", up, shim_mapper, _gpu_plan=getattr(mapper, "_gpu_plan", None))


# ---------------------------------------------------------------------------
# join (operators/__init__.py:2072-2372)
# ---------------------------------------------------------------------------

_LONE_NONE = (None,)
JoinInsertMode = str  # "first" | "last" | "product"
JoinEmitMode = str  # "complete" | "final" | "running"


@dataclass
class _JoinState:
    seen: List[List[Any]]

    @classmethod
    def for_side_count(cls, side_count: int) -> "_JoinState":
        return cls([[] for _ in range(side_count)])

    def set_val(self, side: int, value: Any) -> None:
        self.seen[side] = [value]

    def add_val(self, side: int, value: Any) -> None:
        self.seen[side].append(value)

    def is_set(self, side: int) -> bool:
        return len(self.seen[side]) > 0

    def all_set(self) -> bool:
        return all(len(vals) > 0 for vals in self.seen)

    def astuples(self) -> List[Tuple]:
        return list(itertools.product(*(vals if len(vals) > 0 else _LONE_NONE for vals in self.seen)))

    def clear(self) -> None:
        for vals in self.seen:
            vals.clear()

    def __iadd__(self, other: "_JoinState") -> "_JoinState":
        if len(self.seen) != len(other.seen):
            raise ValueError("join states are not same cardinality")
        self.seen = [x + y for x, y in zip(self.seen, other.seen)]
        return self

    def __ior__(self, other: "_JoinState") -> "_JoinState":
        if len(self.seen) != len(other.seen):
            raise ValueError("join states are not same cardinality")
        self.seen = [y if len(y) > 0 else x for x, y in zip(self.seen, other.seen)]
        return self


@dataclass
class _JoinLogic(StatefulLogic):
    insert_mode: str
    emit_mode: str
    state: _JoinState

    def on_item(self, value):
        side, v = value
        if self.insert_mode == "first" and not self.state.is_set(side):
            self.state.set_val(side, v)
        elif self.insert_mode == "last":
            self.state.set_val(side, v)
        elif self.insert_mode == "product":
            self.state.add_val(side, v)
        if self.emit_mode == "complete" and self.state.all_set():
            return (self.state.astuples(), StatefulLogic.DISCARD)
        if self.emit_mode == "running":
            return (self.state.astuples(), StatefulLogic.RETAIN)
        return (_EMPTY, StatefulLogic.RETAIN)

    def on_eof(self):
        if self.emit_mode == "final":
            return (self.state.astuples(), StatefulLogic.DISCARD)
        return (_EMPTY, StatefulLogic.RETAIN)

    def snapshot(self):
        return copy.deepcopy(self.state)


@operator
def _join_label_merge(step_id: str, *ups: KeyedStream) -> KeyedStream:
    with_labels = [map_value(f"label_{i}", up, partial(lambda i, v: (i, v), i)) for i, up in enumerate(ups)]
    return merge("merge", *with_labels)


@operator
def join(step_id: str, *sides: KeyedStream, insert_mode: str = "last", emit_mode: str = "complete") -> KeyedStream:
    """Gather one value per side for each key (operators/__init__.py:2324)."""
    if insert_mode not in ("first", "last", "product"):
        raise ValueError(f"unknown join insert mode {insert_mode!r}")
    if emit_mode not in ("complete", "final", "running"):
        raise ValueError(f"unknown join emit mode {emit_mode!r}")
    side_count = len(sides)

    def shim_builder(resume_state):
        state = resume_state if resume_state is not None else _JoinState.for_side_count(side_count)
        return _JoinLogic(insert_mode, emit_mode, state)

    merged = _join_label_merge("add_names", *sides)
    plan = None
    if side_count == 2 and insert_mode in ("first", "last"):
        plan = GpuJoinPlan(insert_mode, emit_mode)
    elif 1 <= side_count <= 4:  # (more sides stay on the host engine)
        plan = GpuKeyJoinPlan(insert_mode, emit_mode, side_count)
    return stateful("join", merged, shim_builder, _gpu_plan=plan)
