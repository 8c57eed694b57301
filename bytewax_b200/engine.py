"""Host engine: executes a ``Dataflow`` step tree (the role of ``bytewax._bytewax``).

A small single-process restatement of what the reference's Rust engine does
with the eight core operators (src/worker.rs:255-497, src/operators.rs,
src/inputs.rs, src/outputs.rs; rules collected in SURVEY.md Appendix A):
first data epoch is 1, one ``next_batch`` per partition per activation, one
``mapper(list)`` call per batch, ``stateful_batch`` groups an epoch's items by
key and walks keys in ascending string order, ``on_eof`` once every input is
exhausted, engine errors surface as ``BytewaxRuntimeError`` chained to the
user's exception.  Workers are logical (``worker_count_per_proc`` shards state
by key inside one thread); TCP clusters are out of scope.

Arbitrary Python logic always runs here, on the host.  The one exception is a
``stateful_batch`` whose builder carries a ``GpuFoldPlan`` (numeric windowed
folds made by ``bytewax_b200.operators.windowing``): with the GPU path enabled
(``BYTEWAX_B200_GPU=1`` or ``run_main(..., gpu=True)``) whole epochs are
handed to ``libbwgpu`` instead of calling Python per key.
"""

from __future__ import annotations

import os
import time
from collections import defaultdict
from datetime import datetime, timedelta, timezone
from typing import Any, Dict, List, Optional, Tuple

from bytewax_b200.dataflow import Dataflow, _CoreOperator
from bytewax_b200.errors import BytewaxRuntimeError
from bytewax_b200.inputs import AbortExecution, DynamicSource, FixedPartitionedSource, KeyedColumns
from bytewax_b200.outputs import DynamicSink, FixedPartitionedSink

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
_CORE = {"branch", "flat_map_batch", "input", "inspect_debug", "merge", "output", "redistribute", "stateful_batch", "_noop"}


def _us(dt: datetime) -> int:
    d = dt - EPOCH
    return (d.days * 86400 + d.seconds) * 1_000_000 + d.microseconds


def _dt(us: int) -> datetime:
    return EPOCH + timedelta(microseconds=int(us))


def _route(key: str, workers: int) -> int:
    if workers == 1:
        return 0
    from zlib import crc32

    return crc32(key.encode()) % workers


def _core_steps(flow: Dataflow) -> list:
    out = []

    def walk(steps):
        for st in steps:
            if isinstance(st, _CoreOperator):
                name = type(st).__name__
                if name not in _CORE:
                    raise TypeError(f"Unknown core operator {name!r}")  # src/worker.rs:462-465
                out.append(st)
            else:
                walk(st.substeps)

    walk(flow.substeps)
    return out


def _reraise(msg: str, ex: BaseException):
    if isinstance(ex, KeyboardInterrupt):
        raise ex
    raise BytewaxRuntimeError(msg) from ex


# ---------------------------------------------------------------------------
# GPU-planned windowing step
# ---------------------------------------------------------------------------

_gpu_ctx = None


def _get_gpu_ctx():
    global _gpu_ctx
    if _gpu_ctx is None:
        from bytewax_b200 import gpu

        _gpu_ctx = gpu.Context(int(os.environ.get("BYTEWAX_B200_DEVICE", "0")))
    return _gpu_ctx


class _GpuPlanUnfit(Exception):
    """The first batch of a step whose reducer LOOKED numeric (operator.add, max, min ...) holds values the CUDA fold
    cannot carry (strings, tuples, datetimes, ints beyond int64): the engine runs that step on the host logic instead."""


class _GpuWindowStep:
    """One worker's ``stateful_batch`` of a numeric windowed fold, on ``libbwgpu``."""

    def __init__(self, step_id: str, plan):
        import numpy as np

        from bytewax_b200 import gpu
        from bytewax_b200.operators.windowing import SlidingWindower

        self.np, self.plan, self.step_id = np, plan, step_id
        w = plan.windower
        length = w.length
        offset = w.offset if isinstance(w, SlidingWindower) else w.length
        td_us = lambda td: (td.days * 86400 + td.seconds) * 1_000_000 + td.microseconds  # noqa: E731
        wait = getattr(plan.clock, "wait_for_system_duration", timedelta(0))  # (SystemClock: the watermark IS the system time)
        wait_us = None if wait >= timedelta(days=365 * 200) else td_us(wait)
        self.float_vals = False
        self.fold = None
        self._mk = lambda dtype: gpu.WindowFold(
            _get_gpu_ctx(), plan.reduction, td_us(length), td_us(offset), _us(w.align_to), wait_us, val_dtype=dtype,
            ordered=plan.ordered, capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)),
            max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)), max_emit_rows=1 << 22, max_late_rows=1 << 20)
        self.key_ids: Dict[str, int] = {}
        self.id_keys: Dict[int, str] = {}
        self.resort = False
        self.last_epoch = 0
        self.originals: Dict[int, Any] = {}

    def _key_id(self, k: str) -> int:
        # canonical ASCII decimal text below 2^63: the id is the number itself (str.isdigit alone also accepts other
        # scripts' digits and superscripts); every other key is interned from 2^63 up, so the two ranges never meet
        if k.isascii() and k.isdigit() and (k == "0" or k[0] != "0") and len(k) < 20 and int(k) < (1 << 63):
            return int(k)
        i = self.key_ids.get(k)
        if i is None:
            i = self.key_ids[k] = (1 << 63) + len(self.key_ids)
            self.id_keys[i] = k
            self.resort = True
        return i

    def _key_str(self, i: int) -> str:
        return self.id_keys.get(i) or str(i)

    def on_epoch(self, epoch: int, items: list) -> list:
        np, plan = self.np, self.plan
        keys, ts, vals, orig = [], [], [], []
        cols = [it for it in items if isinstance(it, tuple) and len(it) == 2 and isinstance(it[1], KeyedColumns)]
        if cols and len(cols) != len(items):
            raise TypeError(f"step {self.step_id!r}: mixing KeyedColumns and per-item values in one batch")
        if cols:
            k = np.concatenate([c[1].keys for c in cols]).astype(np.uint64)
            if k.size and int(k.max()) >= (1 << 63):
                raise TypeError(f"step {self.step_id!r}: KeyedColumns keys must be below 2^63 (ids from 2^63 up are interned string keys)")
            t = np.concatenate([c[1].ts_us for c in cols]).astype(np.int64)
            v = None if cols[0][1].vals is None else np.concatenate([c[1].vals for c in cols])
        else:
            getter = getattr(plan.clock, "ts_getter", None)
            if getter is None:  # SystemClock (windowing.py:196-222): an item's timestamp is the system time of its batch
                now_dt = _dt(self._now_us())
                getter = lambda _v: now_dt  # noqa: E731
            for item in items:
                try:
                    key, value = item
                except (TypeError, ValueError) as ex:
                    raise TypeError(f"step {self.step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(item)!r} instead") from ex
                if not isinstance(key, str):
                    raise TypeError(f"step {self.step_id!r} requires `str` keys in `(key, value)` from upstream; got a {type(key)!r} instead")
                keys.append(self._key_id(key))
                ts.append(_us(getter(value)))
                if plan.reduction == "count":
                    vals.append(len(orig))  # the value column carries the arrival index (late rows map back)
                    orig.append(value)
                else:
                    num = plan.value_of(value)
                    if isinstance(num, bool) or not isinstance(num, (int, float)) or (isinstance(num, int) and not -(1 << 63) <= num < (1 << 63)):
                        if self.fold is None:  # nothing folded yet: this step runs on the host logic instead
                            raise _GpuPlanUnfit(f"value {num!r} of type {type(num)!r}")
                        raise TypeError(f"step {self.step_id!r}: the CUDA fold needs numeric values in the int64 / float64 range; got {num!r}")
                    vals.append(num)
            k, t = np.array(keys, dtype=np.uint64), np.array(ts, dtype=np.int64)
            v = np.array(vals) if vals else np.zeros(0, dtype=np.int64)
        if self.fold is None:
            self.float_vals = v is not None and v.dtype.kind == "f"
            self.fold = self._mk("f64" if self.float_vals else "i64")
        if v is not None and v.dtype.kind == "f" and not self.float_vals:
            raise TypeError(f"step {self.step_id!r}: value type changed from integer to float mid-stream")
        self._set_now()
        self.fold.ingest(k, v, t, max(epoch, self.last_epoch))  # (the engine's frontier already keeps epochs in order)
        self.last_epoch = max(epoch, self.last_epoch)
        return self._rows(self.fold.advance(), orig)

    def _now_us(self):
        from bytewax_b200.operators import windowing as W

        if isinstance(self.plan.clock, W.SystemClock):
            return _us(W._get_system_utc())
        getter = getattr(self.plan.clock, "now_getter", None)
        return None if getter is None else _us(getter())

    def _set_now(self):
        # what `before_batch` samples (windowing.py:250-261): the watermark drifts with the system clock
        now = self._now_us()
        if now is not None and now > 0:
            self.fold.set_system_now(now)

    def on_notify(self) -> list:
        """The notify phase (src/operators.rs:808-858): keys whose earliest window's close time has come close what their
        watermark -- which moves with the system clock -- allows, without waiting for another item or EOF."""
        if self.fold is None:
            return []
        now = self._now_us()
        if now is None or now <= 0:
            return []
        return self._rows(self.fold.advance(system_now_us=now), [])

    def on_eof(self) -> list:
        if self.fold is None:
            return []
        out = self._rows(self.fold.eof(), [])
        self.fold.close()
        self.fold = None
        return out

    def release(self):
        """Free the device objects (the engine's cleanup, also after a failed run)."""
        for name in ("fold", "smap", "join"):
            h = getattr(self, name, None)
            if h is not None:
                h.close()
                setattr(self, name, None)

    def _rows(self, em, orig) -> list:
        from bytewax_b200.operators.windowing import WindowColumns, WindowMetadata

        if getattr(self.plan, "columns_out", False) and not self.resort:
            # one item per stream and activation: the library's rows as columns, already in the reference's order
            out = []
            if len(em.late_key):
                out.append(("cols", WindowColumns("L", em.late_key, em.late_window_id, em.late_val)))
            if len(em.closed_key):
                np = self.np
                w = em.closed_window_id
                o, c = self.fold.window_bounds(0)
                off = self.fold.window_bounds(1)[0] - o
                out.append(("cols", WindowColumns("E", em.closed_key, w, em.closed_acc)))
                out.append(("cols", WindowColumns("M", em.closed_key, w, None, o + w.astype(np.int64) * off, c + w.astype(np.int64) * off)))
            return out

        lates = []
        for k, w, val, ep in zip(em.late_key.tolist(), em.late_window_id.tolist(), em.late_val.tolist(), em.late_epoch.tolist()):
            if self.plan.reduction == "count" and orig:
                val = orig[int(val)]
            lates.append((ep, self._key_str(k), w, val))
        if self.resort:
            lates.sort(key=lambda r: (r[0], r[1]))  # stable: arrival order within a key is kept
        rows = [(ks, (w, "L", val)) for _ep, ks, w, val in lates]
        closed = []
        for k, w, acc, ep in zip(em.closed_key.tolist(), em.closed_window_id.tolist(), em.closed_acc.tolist(), em.closed_epoch.tolist()):
            closed.append((ep, self._key_str(k), w, acc))
        if self.resort:
            # interned (non-numeric) keys: restore ascending key-string order per activation; stable
            closed.sort(key=lambda r: (r[0], r[1]))
        for _ep, ks, w, acc in closed:
            o, c = self.fold.window_bounds(w)
            rows.append((ks, (w, "E", acc)))
            rows.append((ks, (w, "M", WindowMetadata(_dt(o), _dt(c)))))
        return rows


class _NoClock:
    def on_notify(self) -> list:
        return []


class _GpuSessionStep(_GpuWindowStep):
    """One worker's ``stateful_batch`` of a numeric fold over a ``SessionWindower`` (``GpuFoldPlan``) on ``bw_session_*``
    (K7): `_WindowLogic` over `_SessionWindowerLogic` (windowing.py:671-810, 1046-1190), one call per activation.  Late
    rows name their input row, so they carry the original item value; ``M`` rows carry the merged session ids."""

    def __init__(self, step_id: str, plan):
        import numpy as np

        self.np, self.plan, self.step_id = np, plan, step_id
        wait = getattr(plan.clock, "wait_for_system_duration", timedelta(0))  # (SystemClock: stamped with the system time, wait 0)
        self.wait_us = None if wait >= timedelta(days=365 * 200) else _td_us(wait)
        self.gap_us = _td_us(plan.windower.gap)
        self.key_ids: Dict[str, int] = {}
        self.id_keys: Dict[int, str] = {}
        self.resort = False
        self.last_epoch = 0
        self.sess = None

    def on_epoch(self, epoch: int, items: list) -> list:
        from bytewax_b200 import gpu

        np, plan = self.np, self.plan
        getter = getattr(plan.clock, "ts_getter", None)
        now = self._now_us()
        if getter is None:  # SystemClock (windowing.py:196-222): an item's timestamp is the system time of its batch
            now_dt = _dt(now)
            getter = lambda _v: now_dt  # noqa: E731
        keys, ts, vals, orig = [], [], [], []
        for item in items:
            key, value = _split_item(self.step_id, item)
            keys.append(self._key_id(key))
            ts.append(_us(getter(value)))
            orig.append(value)
            if plan.reduction != "count":
                num = plan.value_of(value)
                if isinstance(num, bool) or not isinstance(num, (int, float)) or (isinstance(num, int) and not -(1 << 63) <= num < (1 << 63)):
                    if self.sess is None:  # nothing folded yet: this step runs on the host logic instead
                        raise _GpuPlanUnfit(f"value {num!r} of type {type(num)!r}")
                    raise TypeError(f"step {self.step_id!r}: the CUDA session fold needs numeric values in the int64 / float64 range; got {num!r}")
                vals.append(num)
        v = None
        if plan.reduction != "count":
            v = np.array(vals)
            if self.sess is not None and v.dtype.kind == "f" and self.sess.val_dtype != "f64":
                raise TypeError(f"step {self.step_id!r}: value type changed from integer to float mid-stream")
        if self.sess is None:
            self.sess = gpu.SessionFold(
                _get_gpu_ctx(), plan.reduction, self.gap_us, self.wait_us, val_dtype="f64" if v is not None and v.dtype.kind == "f" else "i64",
                capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)), max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)),
                max_emit_rows=1 << 22, max_late_rows=1 << 22, max_sessions_per_key=int(os.environ.get("BYTEWAX_B200_SESSIONS", 64)))
        self.last_epoch = max(epoch, self.last_epoch)
        self.sess.apply(np.array(keys, dtype=np.uint64), v, np.array(ts, dtype=np.int64), self.last_epoch, now or 0)
        return self._session_rows(self.sess.advance(), orig)

    def on_notify(self) -> list:
        if self.sess is None:
            return []
        now = self._now_us()
        if now is None or now <= 0:
            return []
        return self._session_rows(self.sess.advance(system_now_us=now), [])

    def on_eof(self) -> list:
        if self.sess is None:
            return []
        out = self._session_rows(self.sess.eof(), [])
        self.release()
        return out

    def release(self):
        if self.sess is not None:
            self.sess.close()
            self.sess = None

    def _session_rows(self, out, orig) -> list:
        from bytewax_b200.operators.windowing import WindowMetadata

        lates = [(self._key_str(k), orig[r]) for k, r in zip(out.late_key.tolist(), out.late_row.tolist())]
        closed = [(self._key_str(k), i) for i, k in enumerate(out.closed_key.tolist())]
        if self.resort:  # interned (non-numeric) keys: restore ascending key-string order; stable
            lates.sort(key=lambda r: r[0])
            closed.sort(key=lambda r: r[0])
        rows = [(ks, (-1, "L", val)) for ks, val in lates]
        wid, acc = out.closed_window_id.tolist(), out.closed_acc.tolist()
        o, c = out.closed_open_us.tolist(), out.closed_close_us.tolist()
        for ks, i in closed:
            rows.append((ks, (wid[i], "E", acc[i])))
            rows.append((ks, (wid[i], "M", WindowMetadata(_dt(o[i]), _dt(c[i]), set(out.merged(i))))))
        return rows


class _GpuJoinWindowStep(_GpuWindowStep):
    """One worker's ``join_window`` (``GpuJoinWindowPlan``) on ``bw_jwin_*`` (K8): `_WindowLogic` over a tumbling or
    sliding windower with `_JoinWindowLogic` per window (windowing.py:1046-1190, 1849-1902), one call per activation.
    Items are ``(key, (side, value))`` from ``_join_label_merge``; the values stay here, keyed by handle, and each is
    dropped once the device releases its handle.  Late rows carry the labelled item, as on the host."""

    def __init__(self, step_id: str, plan):
        import numpy as np

        self.np, self.plan, self.step_id = np, plan, step_id
        self._windower_spec(plan.windower)
        wait = getattr(plan.clock, "wait_for_system_duration", timedelta(0))  # (SystemClock: stamped with the system time, wait 0)
        self.wait_us = None if wait >= timedelta(days=365 * 200) else _td_us(wait)
        self.key_ids: Dict[str, int] = {}
        self.id_keys: Dict[int, str] = {}
        self.resort = False
        self.last_epoch = 0
        self.values: Dict[int, Any] = {}  # handle -> value, while the device holds the handle
        self.next_handle = 0
        self.jwin = None

    def _windower_spec(self, w):
        from bytewax_b200.operators.windowing import SlidingWindower

        self.length_us = _td_us(w.length)
        self.offset_us = _td_us(w.offset) if isinstance(w, SlidingWindower) else self.length_us
        self.align_us = _us(w.align_to)

    def on_epoch(self, epoch: int, items: list) -> list:
        np, plan = self.np, self.plan
        getter = getattr(plan.clock, "ts_getter", None)
        now = self._now_us()
        if getter is None:  # SystemClock (windowing.py:196-222): an item's timestamp is the system time of its batch
            now_dt = _dt(now)
            getter = lambda _v: now_dt  # noqa: E731
        keys, sides, handles, ts, labelled = [], [], [], [], []
        for item in items:
            key, sv = _split_item(self.step_id, item)
            side, value = sv
            keys.append(self._key_id(key))
            sides.append(side)
            ts.append(_us(getter(value)))
            h = self.next_handle
            self.next_handle += 1
            handles.append(h)
            self.values[h] = value
            labelled.append(sv)
        if self.jwin is None:
            self.jwin = self._make()
        self.last_epoch = max(epoch, self.last_epoch)
        self.jwin.apply(np.array(keys, dtype=np.uint64), np.array(sides, dtype=np.uint8), np.array(handles, dtype=np.uint64),
                        np.array(ts, dtype=np.int64), self.last_epoch, now or 0)
        return self._jwin_rows(self.jwin.advance(), labelled)

    def _make(self):
        from bytewax_b200 import gpu

        plan = self.plan
        return gpu.JoinWindow(
            _get_gpu_ctx(), plan.insert_mode, plan.emit_mode, plan.ordered, plan.sides, self.length_us, self.offset_us, self.align_us,
            self.wait_us, capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)), max_windows_per_key=64,
            max_queued_rows=1 << 22 if plan.ordered else 0, max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)),
            max_emit_rows=1 << 22, max_late_rows=1 << 22)

    def on_notify(self) -> list:
        if self.jwin is None:
            return []
        now = self._now_us()
        if now is None or now <= 0:
            return []
        return self._jwin_rows(self.jwin.advance(system_now_us=now), [])

    def on_eof(self) -> list:
        if self.jwin is None:
            return []
        out = self._jwin_rows(self.jwin.eof(), [])
        self.release()
        return out

    def release(self):
        if self.jwin is not None:
            self.jwin.close()
            self.jwin = None

    def _jwin_rows(self, out, labelled) -> list:
        from bytewax_b200.operators.windowing import WindowMetadata

        V = self.values
        lates = [(self._key_str(k), w, labelled[r]) for k, w, r in zip(out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist())]
        downs = [(self._key_str(k), w, tuple(None if h is None else V[h] for h in t))
                 for k, w, t in zip(out.down_key.tolist(), out.down_window_id.tolist(), out.tuples())]
        metas = [(self._key_str(k), w) for k, w in zip(out.meta_key.tolist(), out.meta_window_id.tolist())]
        if self.resort:  # interned (non-numeric) keys: restore ascending key-string order; stable
            for rows in (lates, downs, metas):
                rows.sort(key=lambda r: r[0])
        rows = [(ks, (w, "L", sv)) for ks, w, sv in lates]
        rows.extend((ks, (w, "E", t)) for ks, w, t in downs)
        for ks, w in metas:
            o, c = self.jwin.window_bounds(w)
            rows.append((ks, (w, "M", WindowMetadata(_dt(o), _dt(c)))))
        for h in out.released.tolist():  # after this call's rows are built: no later row can name these
            del V[h]
        return rows


class _GpuSessionJoinWindowStep(_GpuJoinWindowStep):
    """One worker's ``join_window`` over a ``SessionWindower`` (``GpuJoinWindowPlan``) on ``bw_sjwin_*`` (K10):
    `_WindowLogic` over `_SessionWindowerLogic` with `_JoinWindowLogic` per session (windowing.py:671-810, 1046-1190,
    1849-1902), one call per activation.  Handles, clock sampling, notify, EOF and the key re-sort are the join step's;
    ``M`` rows carry each session's bounds and merged ids from the device, and late rows have window id -1."""

    def _windower_spec(self, w):
        self.gap_us = _td_us(w.gap)

    def _make(self):
        from bytewax_b200 import gpu

        plan = self.plan
        return gpu.SessionJoinWindow(
            _get_gpu_ctx(), plan.insert_mode, plan.emit_mode, plan.ordered, plan.sides, self.gap_us, self.wait_us,
            capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)), max_sessions_per_key=int(os.environ.get("BYTEWAX_B200_SESSIONS", 64)),
            max_queued_rows=1 << 22 if plan.ordered else 0, max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)),
            max_emit_rows=1 << 22, max_late_rows=1 << 22)

    def _jwin_rows(self, out, labelled) -> list:
        from bytewax_b200.operators.windowing import WindowMetadata

        V = self.values
        lates = [(self._key_str(k), labelled[r]) for k, r in zip(out.late_key.tolist(), out.late_row.tolist())]
        downs = [(self._key_str(k), w, tuple(None if h is None else V[h] for h in t))
                 for k, w, t in zip(out.down_key.tolist(), out.down_window_id.tolist(), out.tuples())]
        o, c = out.meta_open_us.tolist(), out.meta_close_us.tolist()
        metas = [(self._key_str(k), w, WindowMetadata(_dt(o[i]), _dt(c[i]), set(out.merged(i))))
                 for i, (k, w) in enumerate(zip(out.meta_key.tolist(), out.meta_window_id.tolist()))]
        if self.resort:  # interned (non-numeric) keys: restore ascending key-string order; stable
            for rows in (lates, downs, metas):
                rows.sort(key=lambda r: r[0])
        rows = [(ks, (-1, "L", sv)) for ks, sv in lates]
        rows.extend((ks, (w, "E", t)) for ks, w, t in downs)
        rows.extend((ks, (w, "M", m)) for ks, w, m in metas)
        for h in out.released.tolist():  # after this call's rows are built: no later row can name these
            del V[h]
        return rows


class _GpuCollectWindowStep(_GpuJoinWindowStep):
    """One worker's ``collect_window`` (``GpuCollectWindowPlan``) on ``bw_collect_*`` (K9): `_WindowLogic` over a tumbling
    or sliding windower with the collect folder per window (windowing.py:1046-1190, 1356-1384, 1436-1576), one call per
    activation.  Handles, clock sampling, notify, EOF and the key re-sort are the join step's; each window's container is
    built here from its handles in play order, with the reference's own folder calls (`append`, `add`, ``d[k] = v``)."""

    def on_epoch(self, epoch: int, items: list) -> list:
        from bytewax_b200 import gpu

        np, plan = self.np, self.plan
        getter = getattr(plan.clock, "ts_getter", None)
        now = self._now_us()
        if getter is None:  # SystemClock (windowing.py:196-222): an item's timestamp is the system time of its batch
            now_dt = _dt(now)
            getter = lambda _v: now_dt  # noqa: E731
        keys, handles, ts, vals = [], [], [], []
        for item in items:
            key, value = _split_item(self.step_id, item)
            self._check_value(value)
            keys.append(self._key_id(key))
            ts.append(_us(getter(value)))
            vals.append(value)
        if self.jwin is None:
            self.jwin = gpu.CollectWindow(
                _get_gpu_ctx(), plan.ordered, self.length_us, self.offset_us, self.align_us, self.wait_us,
                capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)), max_windows_per_key=64,
                max_queued_rows=1 << 22 if plan.ordered else 0, max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)),
                max_emit_rows=1 << 22, max_late_rows=1 << 22)
        for value in vals:
            h = self.next_handle
            self.next_handle += 1
            handles.append(h)
            self.values[h] = value
        self.last_epoch = max(epoch, self.last_epoch)
        self.jwin.apply(np.array(keys, dtype=np.uint64), np.array(handles, dtype=np.uint64), np.array(ts, dtype=np.int64),
                        self.last_epoch, now or 0)
        return self._jwin_rows(self.jwin.advance(), vals)

    def _check_value(self, value):
        # what the folder would reject when it plays the value (windowing.py:1365-1376; `set.add` of an unhashable
        # value): in the first batch the step goes to the host logic, which raises its own error; later, the same error
        # is raised here, at ingest
        try:
            if self.plan.into is dict:
                k, _v = value
                hash(k)
            elif self.plan.into is set:
                hash(value)
        except TypeError as ex:
            if self.jwin is None:
                raise _GpuPlanUnfit(f"value {value!r} of type {type(value)!r}") from ex
            if self.plan.into is dict:
                raise TypeError(f"step {self.plan.step_id!r} collecting into a `dict` requires `(key, value)` 2-tuple as the values in "
                                f"the stream; got a {type(value)!r} instead") from ex
            raise
        except ValueError as ex:
            if self.jwin is None:
                raise _GpuPlanUnfit(f"value {value!r} of type {type(value)!r}") from ex
            raise

    def _container(self, handles):
        V, into = self.values, self.plan.into
        if into is list:
            return [V[h] for h in handles]
        if into is set:
            out = set()
            for h in handles:
                out.add(V[h])
            return out
        d = {}
        for h in handles:
            k, v = V[h]
            d[k] = v
        return d

    def _jwin_rows(self, out, vals) -> list:
        from bytewax_b200.operators.windowing import WindowMetadata

        lates = [(self._key_str(k), w, vals[r]) for k, w, r in zip(out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist())]
        downs = [(self._key_str(k), w, self._container(hs)) for k, w, hs in zip(out.down_key.tolist(), out.down_window_id.tolist(), out.lists())]
        if self.resort:  # interned (non-numeric) keys: restore ascending key-string order; stable
            for rows in (lates, downs):
                rows.sort(key=lambda r: r[0])
        rows = [(ks, (w, "L", v)) for ks, w, v in lates]
        rows.extend((ks, (w, "E", c)) for ks, w, c in downs)
        for ks, w, _c in downs:
            o, c = self.jwin.window_bounds(w)
            rows.append((ks, (w, "M", WindowMetadata(_dt(o), _dt(c)))))
        for h in out.released.tolist():  # after this call's rows are built: no later row can name these
            del self.values[h]
        return rows


def _td_us(td: timedelta) -> int:
    return (td.days * 86400 + td.seconds) * 1_000_000 + td.microseconds


def _gpu_step_for(step_id: str, plan):
    from bytewax_b200.operators import GpuFinalPlan, GpuJoinPlan, GpuSmapPlan
    from bytewax_b200.operators.windowing import GpuCollectWindowPlan, GpuJoinWindowPlan, SessionWindower

    if isinstance(plan, GpuJoinWindowPlan):
        if isinstance(plan.windower, SessionWindower):
            return _GpuSessionJoinWindowStep(step_id, plan)
        return _GpuJoinWindowStep(step_id, plan)
    if isinstance(plan, GpuCollectWindowPlan):
        return _GpuCollectWindowStep(step_id, plan)
    if isinstance(getattr(plan, "windower", None), SessionWindower):
        return _GpuSessionStep(step_id, plan)
    if isinstance(plan, GpuSmapPlan):
        return _GpuSmapStep(step_id, plan)
    if isinstance(plan, GpuJoinPlan):
        return _GpuJoinStep(step_id, plan)
    return _GpuFinalStep(step_id, plan) if isinstance(plan, GpuFinalPlan) else _GpuWindowStep(step_id, plan)


def _split_item(step_id: str, item):
    try:
        key, value = item
    except (TypeError, ValueError) as ex:
        raise TypeError(f"step {step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(item)!r} instead") from ex
    if not isinstance(key, str):
        raise TypeError(f"step {step_id!r} requires `str` keys in `(key, value)` from upstream; got a {type(key)!r} instead")
    return key, value


class _GpuSmapStep(_NoClock, _GpuWindowStep):
    """One worker's ``stateful_map`` with a declared z-score detector (``GpuSmapPlan``) on ``bw_smap_*`` (K5): one call per
    activation instead of one mapper call per item; emits what `_StatefulFlatMapLogic` would, key by key in ascending
    key-string order, a key's items in arrival order (operators/__init__.py:2860-2890, src/operators.rs:755-806)."""

    def __init__(self, step_id: str, plan):
        import numpy as np

        self.np, self.plan, self.step_id = np, plan, step_id
        self.key_ids: Dict[str, int] = {}
        self.id_keys: Dict[int, str] = {}
        self.resort = False
        self.smap = None

    def on_epoch(self, epoch: int, items: list) -> list:
        from bytewax_b200 import gpu

        np = self.np
        keys, vals, names = [], [], []
        for item in items:
            key, value = _split_item(self.step_id, item)
            if isinstance(value, bool) or not isinstance(value, (int, float)):
                if self.smap is None:
                    raise _GpuPlanUnfit(f"value {value!r} of type {type(value)!r}")
                raise TypeError(f"step {self.step_id!r}: the CUDA detector needs float values; got {value!r}")
            keys.append(self._key_id(key))
            names.append(key)
            vals.append(value)
        if self.smap is None:
            self.smap = gpu.ZScoreMap(_get_gpu_ctx(), self.plan.window, self.plan.threshold, val_dtype="f64",
                                      capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)),
                                      max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)))
        mu, sigma, flag = self.smap.apply(np.array(keys, dtype=np.uint64), np.array(vals, dtype=np.float64))
        mu, sigma, flag = mu.tolist(), sigma.tolist(), flag.tolist()
        order = sorted(range(len(items)), key=names.__getitem__)  # stable: arrival order within a key
        return [(names[i], (vals[i], mu[i], sigma[i], flag[i])) for i in order]

    def on_eof(self) -> list:
        if self.smap is not None:
            self.smap.close()
            self.smap = None
        return []


class _GpuJoinStep(_NoClock, _GpuWindowStep):
    """One worker's two-sided ``join`` (``GpuJoinPlan``) on ``bw_join_*`` (K6).  Items are ``(key, (side, value))`` from
    ``_join_label_merge``; the values stay on the host, the device joins their handles (operators/__init__.py:2157-2190)."""

    def __init__(self, step_id: str, plan):
        import numpy as np

        self.np, self.plan, self.step_id = np, plan, step_id
        self.key_ids: Dict[str, int] = {}
        self.id_keys: Dict[int, str] = {}
        self.resort = False
        self.join = None
        self.values: list = []  # handle -> value
        self.last_epoch = 0

    def _rows(self, rows_epochs) -> list:
        rows, epochs = rows_epochs
        out = [(int(ep), self._key_str(k), a, b) for (k, a, b), ep in zip(rows, epochs.tolist())]
        if self.resort:
            out.sort(key=lambda r: (r[0], r[1]))  # interned keys: ascending key-string order per activation; stable
        V = self.values
        return [(ks, (None if a is None else V[a], None if b is None else V[b])) for _ep, ks, a, b in out]

    def on_epoch(self, epoch: int, items: list) -> list:
        from bytewax_b200 import gpu

        np = self.np
        keys, sides, handles = [], [], []
        for item in items:
            key, labelled = _split_item(self.step_id, item)
            side, value = labelled
            keys.append(self._key_id(key))
            sides.append(side)
            handles.append(len(self.values))
            self.values.append(value)
        if self.join is None:
            self.join = gpu.KeyedJoin(_get_gpu_ctx(), self.plan.insert_mode, self.plan.emit_mode,
                                      capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)),
                                      max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)), max_emit_rows=1 << 22)
        self.last_epoch = max(epoch, self.last_epoch)
        self.join.apply(np.array(keys, dtype=np.uint64), np.array(sides, dtype=np.uint8), np.array(handles, dtype=np.uint64), self.last_epoch)
        return self._rows(self.join.advance())

    def on_eof(self) -> list:
        if self.join is None:
            return []
        out = self._rows(self.join.eof())
        self.join.close()
        self.join = None
        return out


class _GpuFinalStep(_NoClock, _GpuWindowStep):
    """One worker's ``stateful_batch`` of a numeric ``*_final`` fold (``reduce_final(add|max|min)``, ``count_final``,
    ``max_final``, ``min_final``) on ``libbwgpu``: ``ts_source == BW_TS_NONE``, every key's accumulator is emitted at EOF in
    ascending key-string order (``_FoldFinalLogic.on_eof`` under the engine's sorted-key EOF walk, src/operators.rs:862-894)."""

    def __init__(self, step_id: str, plan):
        import numpy as np

        from bytewax_b200 import gpu

        self.np, self.plan, self.step_id = np, plan, step_id
        self.float_vals = False
        self.fold = None
        self._mk = lambda dtype: gpu.WindowFold(
            _get_gpu_ctx(), plan.reduction, val_dtype=dtype, final=True,
            capacity_hint=int(os.environ.get("BYTEWAX_B200_KEYS", 1 << 20)),
            max_batch_rows=int(os.environ.get("BYTEWAX_B200_BATCH", 1 << 22)), max_emit_rows=1 << 22, max_late_rows=1 << 10)
        self.key_ids: Dict[str, int] = {}
        self.id_keys: Dict[int, str] = {}
        self.resort = False
        self.last_epoch = 0

    def on_epoch(self, epoch: int, items: list) -> list:
        np = self.np
        keys, vals = [], []
        for item in items:
            try:
                key, value = item
            except (TypeError, ValueError) as ex:
                raise TypeError(f"step {self.step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(item)!r} instead") from ex
            if not isinstance(key, str):
                raise TypeError(f"step {self.step_id!r} requires `str` keys in `(key, value)` from upstream; got a {type(key)!r} instead")
            if isinstance(value, bool) or not isinstance(value, (int, float)) or (isinstance(value, int) and not -(1 << 63) <= value < (1 << 63)):
                if self.fold is None:
                    raise _GpuPlanUnfit(f"value {value!r} of type {type(value)!r}")
                raise TypeError(f"step {self.step_id!r}: the CUDA fold needs numeric values in the int64 / float64 range; got {value!r}")
            keys.append(self._key_id(key))
            vals.append(value)
        if not keys:
            return []
        v = np.array(vals)
        if self.fold is None:
            self.float_vals = v.dtype.kind == "f"
            self.fold = self._mk("f64" if self.float_vals else "i64")
        if v.dtype.kind == "f" and not self.float_vals:
            raise TypeError(f"step {self.step_id!r}: value type changed from integer to float mid-stream")
        self.fold.ingest(np.array(keys, dtype=np.uint64), v, None, max(epoch, self.last_epoch))
        self.last_epoch = max(epoch, self.last_epoch)
        return []

    def on_eof(self) -> list:
        if self.fold is None:
            return []
        em = self.fold.eof()
        self.fold.close()
        self.fold = None
        rows = [(self._key_str(k), acc) for k, acc in zip(em.closed_key.tolist(), em.closed_acc.tolist())]
        if self.resort:
            rows.sort(key=lambda r: r[0])
        return rows


# ---------------------------------------------------------------------------
# the engine proper
# ---------------------------------------------------------------------------


class _InputPart:
    __slots__ = ("part", "worker", "epoch", "started", "eof", "awake_at")

    def __init__(self, part, worker, started):
        self.part, self.worker, self.epoch, self.started, self.eof, self.awake_at = part, worker, 1, started, False, None


class _Run:
    def __init__(self, flow: Dataflow, workers: int, epoch_interval: Optional[timedelta], gpu: Optional[bool]):
        self.flow, self.W = flow, workers
        self.interval = (epoch_interval if epoch_interval is not None else timedelta(seconds=10)).total_seconds()
        self.gpu = gpu if gpu is not None else os.environ.get("BYTEWAX_B200_GPU", "0") == "1"
        self.steps = _core_steps(flow)
        names = [type(s).__name__ for s in self.steps]
        if "input" not in names:
            _reraise("error building Dataflow", ValueError("Dataflow needs to contain at least one input step; add with `bytewax.operators.input`"))
        if "output" not in names and "inspect_debug" not in names:
            _reraise("error building Dataflow", ValueError("Dataflow needs to contain at least one output or inspect step; add with `bytewax.operators.output` or `bytewax.operators.inspect`"))
        seen = set()
        for st in self.steps:
            for name in st.dwn_names:
                port = getattr(st, name)
                for sid in ([port.stream_id] if hasattr(port, "stream_id") else list(port.stream_ids.values())):
                    if sid in seen:
                        raise ValueError(f"duplicate stream ID {sid!r}")
                    seen.add(sid)
        # buffers[stream_id][worker] -> list of (epoch, [items])
        self.buf: Dict[str, List[list]] = defaultdict(lambda: [[] for _ in range(self.W)])
        self.inputs: Dict[str, List[_InputPart]] = {}
        self.sinks: Dict[str, Any] = {}
        self.state: Dict[str, Any] = {}
        self.rr = 0
        self.abort = False

    # -- helpers -------------------------------------------------------------
    def _emit(self, port, worker: int, epoch: int, items: list):
        if items:
            self.buf[port.stream_id][worker].append((epoch, items))

    def _take(self, port) -> List[list]:
        sid = port.stream_id
        if sid not in self.buf:
            return [[] for _ in range(self.W)]
        got = self.buf[sid]
        return got

    # -- per-step execution ----------------------------------------------------
    def _run_input(self, st, now_mono):
        parts = self.inputs.get(st.step_id)
        if parts is None:
            src, parts = st.source, []
            try:
                if isinstance(src, FixedPartitionedSource):
                    for i, name in enumerate(src.list_parts()):
                        parts.append(_InputPart(src.build_part(st.step_id, name, None), i % self.W, now_mono))
                elif isinstance(src, DynamicSource):
                    for w in range(self.W):
                        parts.append(_InputPart(src.build(st.step_id, w, self.W), w, now_mono))
                else:
                    raise TypeError("unknown source type; must subclass `FixedPartitionedSource` or `DynamicSource`")
            except Exception as ex:
                _reraise(f"error building input in step {st.step_id}", ex)
            self.inputs[st.step_id] = parts
        for ip in parts:
            if ip.eof:
                continue
            if ip.awake_at is not None and datetime.now(timezone.utc) < ip.awake_at:
                continue
            try:
                batch = list(ip.part.next_batch())
            except StopIteration:
                ip.eof = True
                batch = None
            except AbortExecution:
                self.abort = True
                return
            except Exception as ex:
                _reraise(f"error calling `next_batch` in step {st.step_id}", ex)
            if batch is not None:
                self._emit(st.down, ip.worker, ip.epoch, batch)
                try:
                    ip.awake_at = ip.part.next_awake()
                except Exception as ex:
                    _reraise(f"error calling `next_awake` in step {st.step_id}", ex)
                if ip.awake_at is None and not batch:
                    ip.awake_at = datetime.now(timezone.utc) + timedelta(milliseconds=1)
            if ip.eof or now_mono - ip.started >= self.interval:
                ip.epoch += 1
                ip.started = now_mono

    def _all_eof(self) -> bool:
        return all(ip.eof for parts in self.inputs.values() for ip in parts) and len(self.inputs) == sum(
            1 for s in self.steps if type(s).__name__ == "input")

    def _run_step(self, st, eof: bool):
        name = type(st).__name__
        if name == "input":
            return
        if name == "flat_map_batch":
            for w, chunks in enumerate(self._take(st.up)):
                for epoch, items in chunks:
                    try:
                        out = st.mapper(items)
                        out = list(out)
                    except Exception as ex:
                        _reraise(f"error calling `mapper` in step {st.step_id}", ex)
                    self._emit(st.down, w, epoch, out)
        elif name == "branch":
            for w, chunks in enumerate(self._take(st.up)):
                for epoch, items in chunks:
                    trues, falses = [], []
                    for item in items:
                        try:
                            keep = st.predicate(item)
                        except Exception as ex:
                            _reraise(f"error calling `predicate` in step {st.step_id}", ex)
                        if not isinstance(keep, bool):
                            _reraise(f"error in step {st.step_id}", TypeError(
                                f"return value of `predicate` in step {st.step_id} must be a `bool`; got a {type(keep)!r} instead"))
                        (trues if keep else falses).append(item)
                    self._emit(st.trues, w, epoch, trues)
                    self._emit(st.falses, w, epoch, falses)
        elif name == "inspect_debug":
            for w, chunks in enumerate(self._take(st.up)):
                for epoch, items in chunks:
                    for item in items:
                        try:
                            st.inspector(st.step_id, item, epoch, w)
                        except Exception as ex:
                            _reraise(f"error calling `inspector` in step {st.step_id}", ex)
                    self._emit(st.down, w, epoch, items)
        elif name == "merge":
            for sid in st.ups.stream_ids.values():
                if sid in self.buf:
                    for w, chunks in enumerate(self.buf[sid]):
                        for epoch, items in chunks:
                            self._emit(st.down, w, epoch, items)
        elif name == "redistribute":
            for w, chunks in enumerate(self._take(st.up)):
                for epoch, items in chunks:
                    per = [[] for _ in range(self.W)]
                    for item in items:
                        per[self.rr % self.W].append(item)
                        self.rr += 1
                    for dw, its in enumerate(per):
                        self._emit(st.down, dw, epoch, its)
        elif name == "output":
            self._run_output(st)
        elif name == "stateful_batch":
            self._run_stateful(st, eof)
        elif name == "_noop":
            for w, chunks in enumerate(self._take(st.up)):
                for epoch, items in chunks:
                    self._emit(st.down, w, epoch, items)

    def _run_output(self, st):
        sink = st.sink
        parts = self.sinks.get(st.step_id)
        if parts is None:
            parts = self.sinks[st.step_id] = {}
        for w, chunks in enumerate(self._take(st.up)):
            for _epoch, items in chunks:
                try:
                    if isinstance(sink, DynamicSink):
                        part = parts.get(w)
                        if part is None:
                            part = parts[w] = sink.build(st.step_id, w, self.W)
                        part.write_batch(items)
                    elif isinstance(sink, FixedPartitionedSink):
                        names = parts.get("__names__")
                        if names is None:
                            names = parts["__names__"] = sink.list_parts()
                        per: Dict[str, list] = defaultdict(list)
                        for item in items:
                            try:
                                key, value = item
                            except (TypeError, ValueError) as ex:
                                raise TypeError(f"step {st.step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(item)!r} instead") from ex
                            if not isinstance(key, str):
                                raise TypeError(f"step {st.step_id!r} requires `str` keys in `(key, value)` from upstream; got a {type(key)!r} instead")
                            per[names[sink.part_fn(key) % len(names)]].append(value)
                        for pname, values in per.items():
                            part = parts.get(pname)
                            if part is None:
                                part = parts[pname] = sink.build_part(st.step_id, pname, None)
                            part.write_batch(values)
                    else:
                        raise TypeError("unknown sink type; must subclass `FixedPartitionedSink` or `DynamicSink`")
                except Exception as ex:
                    _reraise(f"error writing output in step {st.step_id}", ex)

    def _run_stateful(self, st, eof: bool):
        S = self.state.get(st.step_id)
        plan = getattr(st.builder, "_gpu_plan", None) if self.gpu else None
        if S is None:
            S = self.state[st.step_id] = {
                "logics": [dict() for _ in range(self.W)], "sched": [dict() for _ in range(self.W)],
                "gpu": [(_gpu_step_for(st.step_id, plan) if plan is not None else None) for _ in range(self.W)], "eof_done": False,
            }
        # exchange: route every item to the worker owning its key (src/operators.rs:582-591)
        routed: List[Dict[int, list]] = [defaultdict(list) for _ in range(self.W)]
        for _w, chunks in enumerate(self._take(st.up)):
            for epoch, items in chunks:
                for item in items:
                    if isinstance(item, tuple) and len(item) == 2 and isinstance(item[1], KeyedColumns):
                        if plan is not None:
                            routed[0][epoch].append(item)
                        else:
                            # no CUDA path: the rows of the batch as the items the host logic of `fold_columns` folds,
                            # `(str(key), (ts_us, value))`, routed like any other keyed item
                            c = item[1]
                            vals = c.vals.tolist() if c.vals is not None else [1] * len(c)
                            for k, t, v in zip(c.keys.tolist(), c.ts_us.tolist(), vals):
                                ks = str(int(k))
                                routed[_route(ks, self.W)][epoch].append((ks, (int(t), v)))
                        continue
                    try:
                        key, _value = item
                    except (TypeError, ValueError):
                        _reraise(f"error in step {st.step_id}", TypeError(
                            f"step {st.step_id!r} requires `(key, value)` 2-tuple as upstream for routing; got a {type(item)!r} instead"))
                    if not isinstance(key, str):
                        _reraise(f"error in step {st.step_id}", TypeError(
                            f"step {st.step_id!r} requires `str` keys in `(key, value)` from upstream; got a {type(key)!r} instead"))
                    routed[_route(key, self.W)][epoch].append(item)
        now = datetime.now(timezone.utc)
        last_out = S.setdefault("last_out", [0] * self.W)
        # Frontier over the inputs (src/timely.rs:95-133, src/operators.rs:687-728): every input partition advances its
        # own epoch, so an item of epoch e is held back until no partition can still produce an earlier epoch; closed
        # epochs are processed in order and the frontier epoch itself eagerly.  At EOF everything left is flushed.
        pending = S.setdefault("pending", [defaultdict(list) for _ in range(self.W)])
        open_epochs = [ip.epoch for parts in self.inputs.values() for ip in parts if not ip.eof]
        frontier = min(open_epochs) if (open_epochs and not eof) else None
        for w in range(self.W):
            for epoch, items in routed[w].items():
                pending[w][epoch].extend(items)
            ready = {e: pending[w].pop(e) for e in sorted(pending[w]) if frontier is None or e <= frontier}
            g = S["gpu"][w]
            # Epochs of this activation, in order; the epoch of the previous activation is walked again (without items) so
            # that notifications which came due since then fire BEFORE this activation's new items, as the reference does by
            # re-inserting `last_output_epoch` into `process_epochs` (src/operators.rs:698-707, notify phase :808-858).
            epochs = sorted(set(ready) | ({last_out[w]} if last_out[w] else set()))
            last_epoch = 0
            for epoch in epochs:
                last_epoch = epoch
                items = ready.get(epoch)
                if g is not None:
                    if items:
                        try:
                            self._emit(st.down, w, epoch, g.on_epoch(epoch, items))
                        except _GpuPlanUnfit:
                            g = S["gpu"][w] = None  # values the CUDA fold cannot carry: this step stays on the host logic
                        except Exception as ex:
                            _reraise(f"error in the CUDA fold of step {st.step_id}", ex)
                    if g is not None:
                        try:
                            self._emit(st.down, w, epoch, g.on_notify())
                        except Exception as ex:
                            _reraise(f"error in the CUDA fold of step {st.step_id}", ex)
                        continue
                if items:
                    self._host_on_batch(st, S, w, epoch, items)
                self._host_notify(st, S, w, epoch, now)
            if g is None and not epochs:
                self._host_notify(st, S, w, last_epoch, now)
            if last_epoch:
                last_out[w] = last_epoch
            if eof and not S["eof_done"]:
                ep = last_epoch or max((ip.epoch for parts in self.inputs.values() for ip in parts), default=1)
                if g is not None:
                    try:
                        self._emit(st.down, w, ep, g.on_eof())
                    except Exception as ex:
                        _reraise(f"error in the CUDA fold of step {st.step_id}", ex)
                else:
                    self._host_on_eof(st, S, w, ep)
        if eof:
            S["eof_done"] = True

    def _logic_call(self, st, what, key, fn, *a):
        try:
            res = fn(*a)
        except Exception as ex:
            _reraise(f"error calling `StatefulBatchLogic.{what}` in step {st.step_id} for key {key}", ex)
        if what in ("on_batch", "on_notify", "on_eof"):
            try:
                emit, done = res
                emit = list(emit)
            except (TypeError, ValueError) as ex:
                _reraise(f"error in step {st.step_id}", TypeError(
                    f"return value of `{what}` in step {st.step_id} must be a 2-tuple of `(emit, is_complete)`; got a {type(res)!r} instead"))
            if not isinstance(done, bool):
                _reraise(f"error in step {st.step_id}", TypeError(f"`is_complete` in step {st.step_id} must be a `bool`"))
            return emit, done
        return res

    def _host_on_batch(self, st, S, w, epoch, items):
        logics, sched = S["logics"][w], S["sched"][w]
        grouped: Dict[str, list] = {}
        for key, value in items:
            grouped.setdefault(key, []).append(value)
        out, awoken = [], []
        for key in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
            logic = logics.get(key)
            if logic is None:
                try:
                    logic = logics[key] = st.builder(None)
                except Exception as ex:
                    _reraise(f"error calling `builder` in step {st.step_id} for key {key}", ex)
            emit, done = self._logic_call(st, "on_batch", key, logic.on_batch, grouped[key])
            out.extend((key, v) for v in emit)
            if done:
                del logics[key]
                sched.pop(key, None)
            awoken.append(key)
        self._emit(st.down, w, epoch, out)
        for key in awoken:
            logic = logics.get(key)
            if logic is not None:
                at = self._logic_call(st, "notify_at", key, logic.notify_at)
                if at is not None:
                    sched[key] = at

    def _host_notify(self, st, S, w, epoch, now):
        logics, sched = S["logics"][w], S["sched"][w]
        due = sorted(k for k, at in sched.items() if at <= now)
        if not due:
            return
        out = []
        for key in due:
            logic = logics[key]
            emit, done = self._logic_call(st, "on_notify", key, logic.on_notify)
            out.extend((key, v) for v in emit)
            sched.pop(key, None)
            if done:
                del logics[key]
            else:
                at = self._logic_call(st, "notify_at", key, logic.notify_at)
                if at is not None:
                    sched[key] = at
        ep = epoch or max((ip.epoch for parts in self.inputs.values() for ip in parts), default=1)
        self._emit(st.down, w, ep, out)

    def _host_on_eof(self, st, S, w, epoch):
        logics = S["logics"][w]
        out = []
        for key in sorted(logics):  # src/operators.rs:862-894
            emit, done = self._logic_call(st, "on_eof", key, logics[key].on_eof)
            out.extend((key, v) for v in emit)
            if done:
                logics[key] = None
        for key in [k for k, v in logics.items() if v is None]:
            del logics[key]
        self._emit(st.down, w, epoch, out)

    def _next_wakeup(self) -> Optional[datetime]:
        times = [ip.awake_at for parts in self.inputs.values() for ip in parts if not ip.eof and ip.awake_at is not None]
        for S in self.state.values():
            for sched in S["sched"]:
                times.extend(sched.values())
        return min(times) if times else None

    # -- main loop ---------------------------------------------------------------
    def run(self):
        try:
            while True:
                now_mono = time.monotonic()
                for st in self.steps:
                    if type(st).__name__ == "input":
                        self._run_input(st, now_mono)
                        if self.abort:
                            return
                eof = self._all_eof()
                for st in self.steps:
                    self._run_step(st, eof)
                moved = any(chunks for per in self.buf.values() for chunks in per)
                self.buf.clear()
                if eof:
                    return
                if not moved:
                    wake = self._next_wakeup()
                    if wake is not None:
                        delay = (wake - datetime.now(timezone.utc)).total_seconds()
                        if delay > 0:
                            time.sleep(min(delay, 0.05))
        finally:
            for parts in self.inputs.values():
                for ip in parts:
                    try:
                        ip.part.close()
                    except Exception:
                        pass
            for parts in self.sinks.values():
                for name, part in parts.items():
                    if name != "__names__":
                        try:
                            part.close()
                        except Exception:
                            pass
            for S in self.state.values():
                for g in S["gpu"]:
                    if g is not None:
                        g.release()


def run_main(flow: Dataflow, *, epoch_interval: Optional[timedelta] = None, recovery_config=None, gpu: Optional[bool] = None) -> None:
    """Run a dataflow in the calling thread on one worker (src/run.rs:110-119)."""
    if recovery_config is not None:
        raise NotImplementedError("recovery is out of scope of this engine (SURVEY.md section 2 row 12)")
    _Run(flow, 1, epoch_interval, gpu).run()


def cluster_main(flow: Dataflow, addresses: Optional[List[str]], proc_id: int, *, epoch_interval: Optional[timedelta] = None,
                 recovery_config=None, worker_count_per_proc: int = 1, gpu: Optional[bool] = None) -> None:
    """Run with ``worker_count_per_proc`` logical workers in this process (src/run.rs:238-250)."""
    if addresses:
        raise NotImplementedError("multi-process TCP clusters are out of scope; GPUs scale through libbwgpu's exchange")
    if recovery_config is not None:
        raise NotImplementedError("recovery is out of scope of this engine (SURVEY.md section 2 row 12)")
    _Run(flow, max(1, worker_count_per_proc), epoch_interval, gpu).run()


def cli_main(flow: Dataflow, *, workers_per_process: int = 1, process_id: Optional[int] = None, addresses: Optional[List[str]] = None,
             epoch_interval: Optional[timedelta] = None, recovery_config=None) -> None:
    """Entry point of ``python -m bytewax_b200.run`` (src/run.rs:357-394)."""
    if workers_per_process == 1 and not addresses:
        run_main(flow, epoch_interval=epoch_interval, recovery_config=recovery_config)
    else:
        cluster_main(flow, addresses or [], process_id or 0, epoch_interval=epoch_interval, recovery_config=recovery_config,
                     worker_count_per_proc=workers_per_process)
