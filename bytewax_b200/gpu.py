"""Host-side handle on the CUDA windowed-fold path (numpy in, numpy out).

``WindowFold`` is the GPU stand-in for one ``stateful_batch`` step whose logic
is the reference's ``_WindowLogic`` over an ``EventClock`` and a
``SlidingWindower``/``TumblingWindower`` with a numeric fold
(pysrc/bytewax/operators/windowing.py:1046-1190, 1692-1714).  Each
``ingest`` is one activation of src/operators.rs:755-806; ``advance`` returns
what that operator would have given downstream, split like ``WindowOut``
(windowing.py:1193-1222): closed windows (``down`` + ``meta``) and ``late``.
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

from . import _native as N

_NP_VAL = {"u64": np.uint64, "i64": np.int64, "f32": np.float32, "f64": np.float64}


class Context:
    """One rank == one GPU (``bw_ctx``)."""

    def __init__(self, device: int = 0, rank: int = 0, world: int = 1, nccl_id: Optional[bytes] = None):
        self.lib = N.load()
        self.rank, self.world, self.device = rank, world, device
        h = C.c_void_p()
        idbuf = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        N.check(self.lib.bw_ctx_create(device, rank, world, idbuf, C.byref(h)))
        self.h = h

    @classmethod
    def loopback_world(cls, world: int, device: int = 0) -> "list[Context]":
        """``world`` ranks on ONE device, to be driven by one thread each (``bw_loopback_create``): the multi-rank
        path without a second GPU.  The contexts share the world object; closing the last one frees it."""
        lib = N.load()
        w = C.c_void_p()
        N.check(lib.bw_loopback_create(world, C.byref(w)))
        shared = {"handle": w, "open": world}
        out = []
        for r in range(world):
            c = cls.__new__(cls)
            c.lib, c.rank, c.world, c.device = lib, r, world, device
            h = C.c_void_p()
            N.check(lib.bw_ctx_create_loopback(device, r, w, C.byref(h)))
            c.h = h
            c._loop = shared
            out.append(c)
        return out

    @staticmethod
    def new_nccl_id() -> bytes:
        lib = N.load()
        buf = C.create_string_buffer(128)
        N.check(lib.bw_nccl_unique_id(buf))
        return buf.raw

    def close(self):
        if self.h:
            self.lib.bw_ctx_destroy(self.h)
            self.h = None
            loop = getattr(self, "_loop", None)
            if loop is not None:
                loop["open"] -= 1
                if loop["open"] == 0:
                    self.lib.bw_loopback_destroy(loop["handle"])

    # plain device memory (tests / bench)
    def dev_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        N.check(self.lib.bw_dev_alloc(self.h, nbytes, C.byref(p)), self.h)
        return p.value

    def dev_free(self, ptr: int):
        N.check(self.lib.bw_dev_free(self.h, C.c_void_p(ptr)), self.h)

    def h2d(self, dptr: int, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        N.check(self.lib.bw_memcpy(self.h, C.c_void_p(dptr), arr.ctypes.data_as(C.c_void_p), arr.nbytes, 0), self.h)

    def d2h(self, arr: np.ndarray, dptr: int):
        N.check(self.lib.bw_memcpy(self.h, arr.ctypes.data_as(C.c_void_p), C.c_void_p(dptr), arr.nbytes, 1), self.h)

    def flush_l2(self):
        N.check(self.lib.bw_flush_l2(self.h), self.h)


@dataclass
class Emitted:
    """Rows of one ``advance``/``eof`` in the reference's downstream order."""

    closed_key: np.ndarray
    closed_window_id: np.ndarray
    closed_acc: np.ndarray  # typed per reduction / dtype
    closed_count: np.ndarray
    closed_epoch: np.ndarray
    late_key: np.ndarray
    late_window_id: np.ndarray
    late_val: np.ndarray
    late_ts_us: np.ndarray
    late_epoch: np.ndarray

    def down(self, mean: bool = False) -> List[Tuple[int, Tuple[int, object]]]:
        """``(key, (window_id, acc))`` like ``WindowOut.down`` (windowing.py:1196-1200)."""
        if mean:
            return [
                (int(k), (int(w), [float(a), int(c)]))
                for k, w, a, c in zip(self.closed_key, self.closed_window_id, self.closed_acc, self.closed_count)
            ]
        return [(int(k), (int(w), a.item())) for k, w, a in zip(self.closed_key, self.closed_window_id, self.closed_acc)]

    def late(self) -> List[Tuple[int, Tuple[int, object]]]:
        return [(int(k), (int(w), v.item())) for k, w, v in zip(self.late_key, self.late_window_id, self.late_val)]


class WindowFold:
    def __init__(
        self,
        ctx: Context,
        reduction: str = "count",
        length_us: int = 60_000_000,
        offset_us: Optional[int] = None,
        align_to_us: int = 1_640_995_200_000_000,
        wait_us: int = 0,
        val_dtype: str = "u64",
        ts_from_value: bool = False,
        ordered: bool = False,
        emit_order: int = N.ORDER_REFERENCE,
        capacity_hint: int = 1 << 16,
        max_batch_rows: int = 1 << 20,
        max_emit_rows: int = 1 << 20,
        max_late_rows: int = 1 << 16,
        ring_slots: int = 3,
        exchange: int = N.XCHG_P2P,
        final: bool = False,
    ):
        """``final=True``: no event time and no windows -- one accumulator per key, emitted by
        ``eof()`` in key order as window 0 (the ``*_final`` operators); ``ingest`` takes no ``ts``."""
        self.ctx, self.lib = ctx, ctx.lib
        if final:
            ts_from_value, wait_us = False, None
        self.reduction, self.val_dtype, self.ts_from_value = reduction, val_dtype, ts_from_value
        s = N.BwFoldSpec()
        s.struct_size = C.sizeof(N.BwFoldSpec)
        s.reduction = N.RED[reduction]
        s.val_dtype = N.VAL[val_dtype]
        s.ts_source = N.TS_NONE if final else (N.TS_FROM_VALUE if ts_from_value else N.TS_COLUMN)
        s.length_us = length_us
        s.offset_us = offset_us if offset_us is not None else length_us
        s.align_to_us = align_to_us
        s.wait_us = N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.ordered = int(ordered)
        s.emit_order = emit_order
        s.exchange = exchange
        s.ring_slots = ring_slots
        s.capacity_hint = capacity_hint
        s.max_batch_rows = max_batch_rows
        s.max_emit_rows = max_emit_rows
        s.max_late_rows = max_late_rows
        self.spec = s
        self.has_ts = not ts_from_value and not final
        self.has_vals = True
        h = C.c_void_p()
        N.check(self.lib.bw_fold_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    # -- ingest ------------------------------------------------------------
    def acquire(self, rows: Optional[int] = None) -> N.BwBatch:
        b = N.BwBatch()
        n = self.spec.max_batch_rows if rows is None else rows
        N.check(self.lib.bw_ingest_acquire(self.h, n, C.byref(b)), self.ctx.h)
        return b

    def slot_arrays(self, b: N.BwBatch):
        """numpy views on a borrowed pinned slot."""
        cap = int(b.capacity)
        keys = np.ctypeslib.as_array(b.keys, shape=(cap,))
        vals = None
        if b.vals:
            vals = np.ctypeslib.as_array(C.cast(b.vals, C.POINTER(C.c_uint8)), shape=(cap * np.dtype(_NP_VAL[self.val_dtype]).itemsize,)).view(_NP_VAL[self.val_dtype])
        ts = np.ctypeslib.as_array(b.ts_us, shape=(cap,)) if b.ts_us else None
        return keys, vals, ts

    def commit(self, b: N.BwBatch, rows: int, epoch: Optional[int] = None):
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        N.check(self.lib.bw_ingest_commit(self.h, C.byref(b), rows, epoch), self.ctx.h)

    def ingest(self, keys, vals=None, ts=None, epoch: Optional[int] = None):
        """One activation from host arrays (pinned slot -> async H2D -> kernels)."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        n = keys.shape[0]
        b = self.acquire(n)
        k, v, t = self.slot_arrays(b)
        k[:n] = keys
        if self.has_vals:
            if vals is None:
                if self.reduction != "count":
                    raise ValueError("this fold needs a value column")
                v[:n] = 0
            else:
                v[:n] = np.asarray(vals).astype(_NP_VAL[self.val_dtype], copy=False)
        if self.has_ts:
            if ts is None:
                raise ValueError("this fold needs a ts_us column")
            t[:n] = np.asarray(ts, dtype=np.int64)
        self.commit(b, n, epoch)

    def ingest_device(self, d_keys: int, d_vals: Optional[int], d_ts: Optional[int], rows: int, epoch: Optional[int] = None):
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        N.check(
            self.lib.bw_ingest_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_vals or 0), C.c_void_p(d_ts or 0), rows, epoch),
            self.ctx.h,
        )

    def gen_c1(self, d_keys: int, d_vals: int, start: int, rows: int, n_keys: int):
        N.check(self.lib.bw_gen_c1(self.h, C.c_void_p(d_keys), C.c_void_p(d_vals), start, rows, n_keys), self.ctx.h)

    # -- results -----------------------------------------------------------
    def _acc_dtype(self):
        if self.reduction == "count":
            return np.uint64
        if self.reduction == "mean":
            return np.float64
        if self.val_dtype in ("f32", "f64"):
            return np.float64
        return np.int64 if self.val_dtype == "i64" else np.uint64

    def _wrap(self, e: N.BwEmit, copy: bool = True) -> Emitted:
        nc, nl = int(e.n_closed), int(e.n_late)

        def arr(ptr, n, dt):
            if n == 0:
                return np.zeros(0, dtype=dt)
            a = np.ctypeslib.as_array(ptr, shape=(n,)).view(dt)
            return a.copy() if copy else a

        late_dt = np.float64 if self.val_dtype in ("f32", "f64") else (np.int64 if self.val_dtype == "i64" else np.uint64)
        return Emitted(
            arr(e.closed_key, nc, np.uint64), arr(e.closed_window_id, nc, np.int64), arr(e.closed_acc, nc, self._acc_dtype()),
            arr(e.closed_count, nc, np.uint64), arr(e.closed_epoch, nc, np.uint64),
            arr(e.late_key, nl, np.uint64), arr(e.late_window_id, nl, np.int64), arr(e.late_val, nl, late_dt),
            arr(e.late_ts_us, nl, np.int64), arr(e.late_epoch, nl, np.uint64),
        )

    def set_system_now(self, now_us: int):
        """System time of the activations ingested from now on (``bw_fold_set_system_now``; never set: frozen clock)."""
        N.check(self.lib.bw_fold_set_system_now(self.h, int(now_us)), self.ctx.h)

    def advance(self, copy: bool = True, system_now_us: int = 0) -> Emitted:
        """Rows emitted since the last call.  ``copy=False`` returns views of the library's pinned
        output buffers (the C ABI's own contract: valid until the next ``advance``/``eof``).
        ``system_now_us`` > 0 also runs the notify phase at that system time (idle keys' windows close)."""
        e = N.BwEmit()
        N.check(self.lib.bw_advance(self.h, 0, int(system_now_us), C.byref(e)), self.ctx.h)
        return self._wrap(e, copy)

    def eof(self, copy: bool = True) -> Emitted:
        e = N.BwEmit()
        N.check(self.lib.bw_eof(self.h, C.byref(e)), self.ctx.h)
        return self._wrap(e, copy)

    _SNAP_COLS = (("key", np.uint64), ("pane_id", np.int64), ("acc", np.uint64), ("count", np.uint64), ("open_seq", np.uint64),
                  ("max_ts_us", np.int64), ("closed_upto", np.int64))

    def snapshot(self) -> dict:
        """State after the last ``advance`` as numpy columns (one row per live (key, pane)) plus three scalars:
        the columnar form of ``_WindowLogic.snapshot`` (windowing.py:1182-1190) for every key at once."""
        sn = N.BwSnapshot()
        N.check(self.lib.bw_snapshot_take(self.h, C.byref(sn)), self.ctx.h)
        n = int(sn.n)
        out = {name: (np.ctypeslib.as_array(getattr(sn, name), shape=(n,)).view(dt).copy() if n else np.zeros(0, dt))
               for name, dt in self._SNAP_COLS}
        out.update(batch_no=int(sn.batch_no), gmax_ts_us=int(sn.gmax_ts_us), last_epoch=int(sn.last_epoch))
        return out

    def restore(self, snap: dict):
        """Load ``snapshot()`` output into this freshly created fold (same window spec; any capacity / world size)."""
        sn = N.BwSnapshot()
        keep = []
        n = len(snap["key"])
        sn.n = n
        for name, dt in self._SNAP_COLS:
            a = np.ascontiguousarray(snap[name], dtype=dt)
            keep.append(a)
            ctype = C.c_int64 if dt is np.int64 else C.c_uint64
            setattr(sn, name, a.ctypes.data_as(C.POINTER(ctype)))
        sn.batch_no, sn.gmax_ts_us, sn.last_epoch = snap["batch_no"], snap["gmax_ts_us"], snap["last_epoch"]
        N.check(self.lib.bw_snapshot_load(self.h, C.byref(sn)), self.ctx.h)
        self._epoch = max(self._epoch, int(snap["last_epoch"]))

    def window_bounds(self, window_id: int) -> Tuple[int, int]:
        o, c = C.c_int64(), C.c_int64()
        self.lib.bw_window_bounds(C.byref(self.spec), window_id, C.byref(o), C.byref(c))
        return o.value, c.value

    def stats(self) -> N.BwStats:
        st = N.BwStats()
        N.check(self.lib.bw_fold_stats(self.h, C.byref(st)), self.ctx.h)
        return st

    def reset_timers(self):
        N.check(self.lib.bw_fold_reset_timers(self.h), self.ctx.h)

    def time_begin(self):
        N.check(self.lib.bw_fold_time_begin(self.h), self.ctx.h)

    def time_end(self) -> float:
        ms = C.c_float()
        N.check(self.lib.bw_fold_time_end(self.h, C.byref(ms)), self.ctx.h)
        return ms.value

    def sync(self):
        N.check(self.lib.bw_fold_sync(self.h), self.ctx.h)

    def set_segfold_parts(self, parts: int):
        """Measurement: which parts of the segment fold run (``bw_fold_set_segfold_parts``)."""
        N.check(self.lib.bw_fold_set_segfold_parts(self.h, parts), self.ctx.h)

    def check_key_column(self) -> Tuple[int, int]:
        """(slots whose dense key differs from the hot slot's key, slots holding a key), after the work in flight."""
        bad, used = C.c_uint64(), C.c_uint64()
        N.check(self.lib.bw_fold_check_key_column(self.h, C.byref(bad), C.byref(used)), self.ctx.h)
        return bad.value, used.value

    def close(self):
        if self.h:
            self.lib.bw_fold_destroy(self.h)
            self.h = None


class ZScoreMap:
    """``stateful_map`` with the rolling z-score detector (``bw_smap``; examples/anomaly_detector.py:16-48).

    On a multi-rank context (``world > 1``) the map is rank-local unless ``shard_by_key=True``: each rank keeps its own
    ring for every key it sees, so the caller must send every row of a key to one rank.  With ``shard_by_key=True`` it is
    sharded by key and collective: every rank creates it with the same arguments and calls ``apply`` or ``apply_device``
    once per activation, with its own rows (possibly none).  Each row goes to rank ``bw_route(key, world)``, which maps
    what arrived in (source rank, source order) and sends each row's results back, so a rank's outputs stay aligned with
    its own input rows; every rank's outputs concatenated rank-major equal a world-1 map over the rank-major
    concatenation of every rank's rows.  A call one rank cannot make (too many rows, a NULL column, a failed map) fails
    on every rank, and no rank maps it; a full key table on an owner fails the call on every rank and the map refuses
    every later call.  Close it only once no rank calls it any more."""

    def __init__(self, ctx: Context, window: int = 10, threshold: float = 2.0, val_dtype: str = "f32", capacity_hint: int = 1 << 16,
                 max_batch_rows: int = 1 << 20, shard_by_key: bool = False):
        self.ctx, self.lib, self.val_dtype = ctx, ctx.lib, val_dtype
        s = N.BwSmapSpec()
        s.struct_size = C.sizeof(N.BwSmapSpec)
        s.window, s.val_dtype, s.threshold = window, N.VAL[val_dtype], threshold
        s.capacity_hint, s.max_batch_rows = capacity_hint, max_batch_rows
        s.shard_by_key = int(shard_by_key)
        h = C.c_void_p()
        N.check(self.lib.bw_smap_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h

    def apply(self, keys, vals):
        """One activation -> (mu f64[n], sigma f64[n], anomalous bool[n]) aligned with the input rows."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        vals = np.ascontiguousarray(vals, dtype=_NP_VAL[self.val_dtype])
        n = keys.shape[0]
        mu, sigma, flag = np.empty(n, np.float64), np.empty(n, np.float64), np.empty(n, np.uint8)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_smap_apply(self.h, vp(keys), vp(vals), n, vp(mu), vp(sigma), vp(flag)), self.ctx.h)
        return mu, sigma, flag.astype(bool)

    def apply_device(self, d_keys: int, d_vals: int, rows: int, d_mu: int, d_sigma: int, d_flag: int):
        """One activation from device columns (u64 keys, f32 / f64 values) into device columns (f64 mu, f64 sigma, u8
        flag), aligned with the input rows.  On one rank it returns once the work is enqueued (``sync`` waits); sharded
        by key it returns once the call is complete."""
        N.check(self.lib.bw_smap_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_vals), rows, C.c_void_p(d_mu),
                                              C.c_void_p(d_sigma), C.c_void_p(d_flag)), self.ctx.h)

    def sync(self):
        N.check(self.lib.bw_smap_sync(self.h), self.ctx.h)

    def close(self):
        if self.h:
            self.lib.bw_smap_destroy(self.h)
            self.h = None


class KeyedJoin:
    """Two-sided keyed join (``bw_join``; operators/__init__.py:2157-2190).

    On a multi-rank context (``world > 1``) the join is sharded by key and collective: every rank creates it with the
    same arguments and calls ``apply`` once per activation, with its own rows (possibly none) and the same epoch.  Each
    row goes to rank ``bw_route(key, world)``, which joins what arrived in (source rank, source order); ``vals`` is an
    opaque u64 payload that travels with its row.  A rank's ``advance`` / ``eof`` return the rows of the keys it owns.
    An ``apply`` that cannot go ahead on one rank (more than ``max_batch_rows`` rows, a NULL column, an epoch below the
    last one since that rank's last ``advance``) still takes part in the exchange: that rank raises its own error, every
    other rank ``BW_ERR_STATE``, no rank plays the call, and the next call goes on as if it had not been made.  A full
    key table or emit buffer raises on its owner's ``advance``, as on one GPU; the other ranks' keys stay exact.  Close
    it only once no rank calls it any more."""

    INSERT = {"first": 0, "last": 1}
    EMIT = {"complete": 0, "final": 1, "running": 2}

    def __init__(self, ctx: Context, insert_mode: str = "last", emit_mode: str = "complete", capacity_hint: int = 1 << 16,
                 max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20):
        self.ctx, self.lib = ctx, ctx.lib
        s = N.BwJoinSpec()
        s.struct_size = C.sizeof(N.BwJoinSpec)
        s.insert_mode, s.emit_mode = self.INSERT[insert_mode], self.EMIT[emit_mode]
        s.capacity_hint, s.max_batch_rows, s.max_emit_rows = capacity_hint, max_batch_rows, max_emit_rows
        h = C.c_void_p()
        N.check(self.lib.bw_join_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def apply(self, keys, sides, vals, epoch: Optional[int] = None):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        sides = np.ascontiguousarray(sides, dtype=np.uint8)
        vals = np.ascontiguousarray(vals, dtype=np.uint64)
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_join_apply(self.h, vp(keys), vp(sides), vp(vals), keys.shape[0], epoch), self.ctx.h)

    def _rows(self, r: N.BwJoinRows):
        n = int(r.n)

        def arr(ptr):
            return np.ctypeslib.as_array(ptr, shape=(n,)).copy() if n else np.zeros(0, np.uint64)

        key, l, rr, mask, epoch = arr(r.key), arr(r.left), arr(r.right), arr(r.mask), arr(r.epoch)
        rows = [(int(k), int(a) if m & 1 else None, int(b) if m & 2 else None) for k, a, b, m in zip(key, l, rr, mask)]
        return rows, epoch

    def advance(self):
        """Rows ``(key, left_or_None, right_or_None)`` emitted since the last call, in the reference's order."""
        r = N.BwJoinRows()
        N.check(self.lib.bw_join_advance(self.h, C.byref(r)), self.ctx.h)
        return self._rows(r)

    def eof(self):
        r = N.BwJoinRows()
        N.check(self.lib.bw_join_eof(self.h, C.byref(r)), self.ctx.h)
        return self._rows(r)

    def close(self):
        if self.h:
            self.lib.bw_join_destroy(self.h)
            self.h = None


@dataclass
class SessionRows:
    """Rows of one ``SessionFold.advance`` / ``eof`` in the reference's downstream order."""

    closed_key: np.ndarray
    closed_window_id: np.ndarray
    closed_acc: np.ndarray  # uint64 (count), int64 or float64
    closed_open_us: np.ndarray
    closed_close_us: np.ndarray
    closed_epoch: np.ndarray
    merged_off: np.ndarray  # [n_closed + 1] into merged_ids
    merged_ids: np.ndarray
    late_key: np.ndarray
    late_epoch: np.ndarray
    late_activation: np.ndarray
    late_row: np.ndarray  # the row's index in the columns its source rank passed
    late_rank: np.ndarray  # that source rank; all zeros on one rank

    def merged(self, i: int) -> List[int]:
        return self.merged_ids[self.merged_off[i] : self.merged_off[i + 1]].tolist()

    def rows(self) -> list:
        """``[key, window_id, tag, payload]`` rows like the reference's window events: per closed session ``E`` (the
        accumulator) then ``M`` (``[open_us, close_us, merged ids]``); late rows (``L``, window -1) carry the input
        position ``(activation, row)`` as payload."""
        out = []
        for i, (k, w, a, o, c) in enumerate(zip(self.closed_key.tolist(), self.closed_window_id.tolist(), self.closed_acc.tolist(),
                                               self.closed_open_us.tolist(), self.closed_close_us.tolist())):
            out.append([k, w, "E", a])
            out.append([k, w, "M", [o, c, self.merged(i)]])
        out.extend([k, -1, "L", (a, r)] for k, a, r in zip(self.late_key.tolist(), self.late_activation.tolist(), self.late_row.tolist()))
        return out


class SessionFold:
    """Session-window count / sum / min / max by key (``bw_session``, K7; windowing.py:671-810, 1046-1190).

    On a multi-rank context (``world > 1``) the fold needs ``shard_by_key=True`` (without it, create raises, as a fold
    that cannot see the other ranks' rows would be wrong); it is then sharded by key and collective: every rank creates
    it with the same arguments and calls ``apply`` or ``apply_device`` once per activation, with its own rows (possibly none), the
    same epoch and the same ``system_now_us``.  Each row goes to rank ``bw_route(key, world)``, which folds what arrived
    in (source rank, source order).  A call one rank cannot make (too many rows, a decreasing epoch, a failed fold)
    fails on every rank, and no rank folds it.  A rank's ``advance`` / ``eof`` return the sessions and late rows of the
    keys it owns; a late row names its input row by (``late_activation``, ``late_rank``, ``late_row``).  Close it only
    once no rank calls it any more."""

    def __init__(self, ctx: Context, reduction: str = "count", gap_us: int = 10_000_000, wait_us: Optional[int] = 0,
                 val_dtype: str = "i64", capacity_hint: int = 1 << 16, max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20,
                 max_late_rows: int = 1 << 20, max_sessions_per_key: int = 16, shard_by_key: bool = False):
        """``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``)."""
        self.ctx, self.lib = ctx, ctx.lib
        self.reduction, self.val_dtype = reduction, val_dtype
        s = N.BwSessionSpec()
        s.struct_size = C.sizeof(N.BwSessionSpec)
        s.reduction, s.val_dtype = N.RED[reduction], N.VAL[val_dtype]
        s.gap_us, s.wait_us = gap_us, N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_batch_rows, s.max_emit_rows, s.max_late_rows = capacity_hint, max_batch_rows, max_emit_rows, max_late_rows
        s.max_sessions_per_key = max_sessions_per_key
        s.shard_by_key = int(shard_by_key)
        self.spec = s
        h = C.c_void_p()
        N.check(self.lib.bw_session_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def apply(self, keys, vals, ts_us, epoch: Optional[int] = None, system_now_us: int = 0):
        """One activation from host arrays (``vals`` may be None for count).  ``system_now_us``: ``now_getter()``."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        ts = np.ascontiguousarray(ts_us, dtype=np.int64)
        v = None if vals is None else np.ascontiguousarray(vals, dtype=_NP_VAL[self.val_dtype])
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_session_apply(self.h, vp(keys), None if v is None else vp(v), vp(ts), keys.shape[0], epoch,
                                          int(system_now_us)), self.ctx.h)

    def apply_device(self, d_keys: int, d_vals: Optional[int], d_ts: int, rows: int, epoch: Optional[int] = None, system_now_us: int = 0):
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        N.check(self.lib.bw_session_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_vals or 0), C.c_void_p(d_ts), rows, epoch,
                                                 int(system_now_us)), self.ctx.h)

    def _wrap(self, r: N.BwSessionRows) -> SessionRows:
        nc, nl = int(r.n_closed), int(r.n_late)

        def arr(ptr, n, dt):
            return np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).copy() if n else np.zeros(0, dt)

        if self.reduction == "count":
            acc_dt = np.uint64
        else:
            acc_dt = np.float64 if self.val_dtype == "f64" else np.int64
        off = arr(r.merged_off, nc + 1, np.uint64).astype(np.int64)
        return SessionRows(arr(r.closed_key, nc, np.uint64), arr(r.closed_window_id, nc, np.int64), arr(r.closed_acc, nc, acc_dt),
                           arr(r.closed_open_us, nc, np.int64), arr(r.closed_close_us, nc, np.int64), arr(r.closed_epoch, nc, np.uint64),
                           off, arr(r.merged_ids, int(off[-1]), np.int64),
                           arr(r.late_key, nl, np.uint64), arr(r.late_epoch, nl, np.uint64), arr(r.late_activation, nl, np.uint64),
                           arr(r.late_row, nl, np.uint64), arr(r.late_rank, nl, np.uint64))

    def advance(self, system_now_us: int = 0) -> SessionRows:
        """Rows since the last call; ``system_now_us`` > 0 first runs the notify phase at that system time."""
        r = N.BwSessionRows()
        N.check(self.lib.bw_session_advance(self.h, int(system_now_us), C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self) -> SessionRows:
        r = N.BwSessionRows()
        N.check(self.lib.bw_session_eof(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self.lib.bw_session_destroy(self.h)
            self.h = None


@dataclass
class JoinWindowRows:
    """Rows of one ``JoinWindow.advance`` / ``eof``, each stream in the reference's downstream order, and the handles
    released since the previous one."""

    down_key: np.ndarray
    down_window_id: np.ndarray
    down_handles: np.ndarray  # [rows, sides] uint64; valid where the side's bit of down_mask is set
    down_mask: np.ndarray
    down_epoch: np.ndarray
    meta_key: np.ndarray
    meta_window_id: np.ndarray
    meta_epoch: np.ndarray
    late_key: np.ndarray
    late_window_id: np.ndarray
    late_epoch: np.ndarray
    late_activation: np.ndarray
    late_row: np.ndarray  # the row's index in the columns its source rank passed
    late_rank: np.ndarray  # that source rank; all zeros on one rank
    released: np.ndarray  # uint64, in no particular order

    def tuples(self) -> List[tuple]:
        """The joined tuple of every down row: a handle per side, None where the side is unset."""
        m = self.down_mask.tolist()
        return [tuple(int(h[s]) if mk >> s & 1 else None for s in range(len(h))) for h, mk in zip(self.down_handles.tolist(), m)]


class _HandleJoin:
    """What the handle joins `JoinWindow` (``bw_jwin_*``) and `SessionJoinWindow` (``bw_sjwin_*``) share: their modes,
    epochs, and the apply / advance / eof / close calls, which differ only in the C prefix and the rows they wrap."""

    INSERT = {"first": 0, "last": 1}
    EMIT = {"complete": 0, "final": 1, "running": 2}
    _PREFIX = ""  # the C ABI prefix
    _ROWS = None  # its rows struct

    def _create(self, ctx: Context, spec, sides: int):
        self.ctx, self.lib, self.sides, self.spec = ctx, ctx.lib, sides, spec
        h = C.c_void_p()
        N.check(self._fn("create")(ctx.h, C.byref(spec), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def _fn(self, name: str):
        return getattr(self.lib, f"{self._PREFIX}_{name}")

    def _next_epoch(self, epoch: Optional[int]) -> int:
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        return epoch

    def apply(self, keys, sides, handles, ts_us, epoch: Optional[int] = None, system_now_us: int = 0):
        """One activation from host arrays.  ``system_now_us``: ``now_getter()`` of the activation."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        sides = np.ascontiguousarray(sides, dtype=np.uint8)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        ts = np.ascontiguousarray(ts_us, dtype=np.int64)
        epoch = self._next_epoch(epoch)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self._fn("apply")(self.h, vp(keys), vp(sides), vp(handles), vp(ts), keys.shape[0], epoch, int(system_now_us)), self.ctx.h)

    def apply_device(self, d_keys: int, d_sides: int, d_handles: int, d_ts: int, rows: int, epoch: Optional[int] = None,
                     system_now_us: int = 0):
        epoch = self._next_epoch(epoch)
        N.check(self._fn("apply_device")(self.h, C.c_void_p(d_keys), C.c_void_p(d_sides), C.c_void_p(d_handles), C.c_void_p(d_ts),
                                         rows, epoch, int(system_now_us)), self.ctx.h)

    def advance(self, system_now_us: int = 0):
        """Rows since the last call; ``system_now_us`` > 0 first runs the notify phase at that system time."""
        r = self._ROWS()
        N.check(self._fn("advance")(self.h, int(system_now_us), C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self):
        r = self._ROWS()
        N.check(self._fn("eof")(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self._fn("destroy")(self.h)
            self.h = None


class JoinWindow(_HandleJoin):
    """``join_window`` with insert mode first / last over tumbling or sliding windows (``bw_jwin``, K8;
    windowing.py:1046-1190, 1849-1902).  Values travel as uint64 handles; the caller keeps the objects and may drop
    each one once it comes back in ``released``.

    On a multi-rank context (``world > 1``) the join needs ``shard_by_key=True`` (without it, create raises, as a join
    that cannot see the other ranks' rows would be wrong); it is then sharded by key and collective: every rank creates
    it with the same arguments and calls ``apply`` or ``apply_device`` once per activation, with its own rows (possibly
    none), the same epoch and the same ``system_now_us``.  Each row goes to rank ``bw_route(key, world)``, which joins
    what arrived in (source rank, source order).  A call one rank cannot make (too many rows, a side out of range, a
    decreasing epoch, a failed join) fails on every rank, and no rank plays it.  A rank's ``advance`` / ``eof`` return
    the rows of the keys it owns, and ``released`` lists each handle once, on the owner of its key (handles travel
    opaquely: put the source rank in the handle if it is needed); a late row names its input row by
    (``late_activation``, ``late_rank``, ``late_row``).  Close it only once no rank calls it any more."""

    _PREFIX, _ROWS = "bw_jwin", N.BwJwinRows

    def __init__(self, ctx: Context, insert_mode: str = "last", emit_mode: str = "final", ordered: bool = True, sides: int = 2,
                 length_us: int = 10_000_000, offset_us: Optional[int] = None, align_us: int = 0, wait_us: Optional[int] = 0,
                 capacity_hint: int = 1 << 16, max_windows_per_key: int = 16, max_queued_rows: int = 1 << 20,
                 max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20, max_late_rows: int = 1 << 20, shard_by_key: bool = False):
        """``offset_us=None``: tumbling.  ``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``)."""
        s = N.BwJwinSpec()
        s.struct_size = C.sizeof(N.BwJwinSpec)
        s.insert_mode, s.emit_mode = self.INSERT.get(insert_mode, -1), self.EMIT.get(emit_mode, -1)
        s.ordered, s.sides, s.max_windows_per_key = int(ordered), sides, max_windows_per_key
        s.length_us, s.offset_us, s.align_us = length_us, length_us if offset_us is None else offset_us, align_us
        s.wait_us = N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_queued_rows, s.max_batch_rows = capacity_hint, max_queued_rows, max_batch_rows
        s.max_emit_rows, s.max_late_rows = max_emit_rows, max_late_rows
        s.shard_by_key = int(shard_by_key)
        self._create(ctx, s, sides)

    def window_bounds(self, window_id: int):
        """``(open_us, close_us)`` of a window (windowing.py:620-623)."""
        o = self.spec.align_us + self.spec.offset_us * window_id
        return o, o + self.spec.length_us

    def _wrap(self, r: N.BwJwinRows) -> JoinWindowRows:
        nd, nm, nl, nr = int(r.n_down), int(r.n_meta), int(r.n_late), int(r.n_released)

        def arr(ptr, n, dt=np.uint64):
            return np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).copy() if n else np.zeros(0, dt)

        hs = np.stack([arr(r.down_handle[s], nd) for s in range(self.sides)], axis=1) if nd else np.zeros((0, self.sides), np.uint64)
        return JoinWindowRows(arr(r.down_key, nd), arr(r.down_window_id, nd, np.int64), hs, arr(r.down_mask, nd), arr(r.down_epoch, nd),
                              arr(r.meta_key, nm), arr(r.meta_window_id, nm, np.int64), arr(r.meta_epoch, nm),
                              arr(r.late_key, nl), arr(r.late_window_id, nl, np.int64), arr(r.late_epoch, nl),
                              arr(r.late_activation, nl), arr(r.late_row, nl), arr(r.late_rank, nl), arr(r.released, nr))


class ProductJoinWindow(JoinWindow):
    """``join_window`` with insert mode product over tumbling or sliding windows (``bw_pjwin``, K14;
    windowing.py:1046-1190, 1849-1902, ``_JoinState`` operators/__init__.py:2072-2120).  Each down row is one tuple of an
    emission's ``itertools.product``, expanded on the device; values travel as uint64 handles, and each comes back in
    ``released`` once no window list and no queue entry holds it."""

    _PREFIX, _ROWS = "bw_pjwin", N.BwJwinRows

    def __init__(self, ctx: Context, emit_mode: str = "final", ordered: bool = True, sides: int = 2, length_us: int = 10_000_000,
                 offset_us: Optional[int] = None, align_us: int = 0, wait_us: Optional[int] = 0, capacity_hint: int = 1 << 16,
                 max_windows_per_key: int = 16, max_queued_rows: int = 1 << 20, max_batch_rows: int = 1 << 20,
                 max_emit_rows: int = 1 << 20, max_late_rows: int = 1 << 20, max_product_rows: int = 1 << 26):
        """``offset_us=None``: tumbling.  ``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``).
        ``max_product_rows``: down rows one ``advance`` / ``eof`` may hand out."""
        s = N.BwPjwinSpec()
        s.struct_size = C.sizeof(N.BwPjwinSpec)
        s.emit_mode = self.EMIT.get(emit_mode, -1)
        s.ordered, s.sides, s.max_windows_per_key = int(ordered), sides, max_windows_per_key
        s.length_us, s.offset_us, s.align_us = length_us, length_us if offset_us is None else offset_us, align_us
        s.wait_us = N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_queued_rows, s.max_batch_rows = capacity_hint, max_queued_rows, max_batch_rows
        s.max_emit_rows, s.max_late_rows, s.max_product_rows = max_emit_rows, max_late_rows, max_product_rows
        self._create(ctx, s, sides)


@dataclass
class SessionJoinWindowRows(JoinWindowRows):
    """Rows of one ``SessionJoinWindow.advance`` / ``eof``: the join's streams, with each meta row's session bounds and
    merged ids.  Late rows all have window id -1 (``LATE_SESSION_ID``)."""

    meta_open_us: np.ndarray = None
    meta_close_us: np.ndarray = None
    merged_off: np.ndarray = None  # [n_meta + 1] into merged_ids
    merged_ids: np.ndarray = None

    def merged(self, i: int) -> List[int]:
        """The ids merged directly into meta row ``i``'s session, ascending."""
        return self.merged_ids[self.merged_off[i] : self.merged_off[i + 1]].tolist()


class SessionJoinWindow(_HandleJoin):
    """``join_window`` with insert mode first / last over session windows (``bw_sjwin``, K10; windowing.py:671-810,
    1046-1190, 1849-1902).  Values travel as uint64 handles; the caller keeps the objects and may drop each one once it
    comes back in ``released``.  Session bounds come with each meta row."""

    _PREFIX, _ROWS = "bw_sjwin", N.BwSjwinRows

    def __init__(self, ctx: Context, insert_mode: str = "last", emit_mode: str = "final", ordered: bool = True, sides: int = 2,
                 gap_us: int = 10_000_000, wait_us: Optional[int] = 0, capacity_hint: int = 1 << 16, max_sessions_per_key: int = 16,
                 max_queued_rows: int = 1 << 20, max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20, max_late_rows: int = 1 << 20):
        """``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``)."""
        s = N.BwSjwinSpec()
        s.struct_size = C.sizeof(N.BwSjwinSpec)
        s.insert_mode, s.emit_mode = self.INSERT.get(insert_mode, -1), self.EMIT.get(emit_mode, -1)
        s.ordered, s.sides, s.max_sessions_per_key = int(ordered), sides, max_sessions_per_key
        s.gap_us, s.wait_us = gap_us, N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_queued_rows, s.max_batch_rows = capacity_hint, max_queued_rows, max_batch_rows
        s.max_emit_rows, s.max_late_rows = max_emit_rows, max_late_rows
        self._create(ctx, s, sides)

    def _wrap(self, r: N.BwSjwinRows) -> SessionJoinWindowRows:
        nd, nm, nl, nr = int(r.n_down), int(r.n_meta), int(r.n_late), int(r.n_released)

        def arr(ptr, n, dt=np.uint64):
            return np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).copy() if n else np.zeros(0, dt)

        hs = np.stack([arr(r.down_handle[s], nd) for s in range(self.sides)], axis=1) if nd else np.zeros((0, self.sides), np.uint64)
        off = arr(r.merged_off, nm + 1).astype(np.int64)
        # by keyword: the fields of JoinWindowRows come first (K10 runs on one GPU: its late rows' source rank is 0)
        return SessionJoinWindowRows(down_key=arr(r.down_key, nd), down_window_id=arr(r.down_window_id, nd, np.int64), down_handles=hs,
                                     down_mask=arr(r.down_mask, nd), down_epoch=arr(r.down_epoch, nd), meta_key=arr(r.meta_key, nm),
                                     meta_window_id=arr(r.meta_window_id, nm, np.int64), meta_epoch=arr(r.meta_epoch, nm),
                                     late_key=arr(r.late_key, nl), late_window_id=np.full(nl, -1, np.int64), late_epoch=arr(r.late_epoch, nl),
                                     late_activation=arr(r.late_activation, nl), late_row=arr(r.late_row, nl),
                                     late_rank=np.zeros(nl, np.uint64), released=arr(r.released, nr),
                                     meta_open_us=arr(r.meta_open_us, nm, np.int64), meta_close_us=arr(r.meta_close_us, nm, np.int64),
                                     merged_off=off, merged_ids=arr(r.merged_ids, int(off[-1]), np.int64))


class SessionProductJoinWindow(SessionJoinWindow):
    """``join_window`` with insert mode product over session windows (``bw_spjwin``, K16; windowing.py:671-810,
    1046-1190, 1849-1902, ``_JoinState`` operators/__init__.py:2072-2120).  Each down row is one tuple of an emission's
    ``itertools.product``, expanded on the device; a merge appends the merged-away session's lists to the survivor's.
    Values travel as uint64 handles, and each comes back in ``released`` once no session list and no queue entry holds
    it.  Session bounds and merged ids come with each meta row."""

    _PREFIX, _ROWS = "bw_spjwin", N.BwSjwinRows

    def __init__(self, ctx: Context, emit_mode: str = "final", ordered: bool = True, sides: int = 2, gap_us: int = 10_000_000,
                 wait_us: Optional[int] = 0, capacity_hint: int = 1 << 16, max_sessions_per_key: int = 16, max_queued_rows: int = 1 << 20,
                 max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20, max_late_rows: int = 1 << 20,
                 max_product_rows: int = 1 << 26):
        """``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``).  ``max_product_rows``: down rows
        one ``advance`` / ``eof`` may hand out."""
        s = N.BwSpjwinSpec()
        s.struct_size = C.sizeof(N.BwSpjwinSpec)
        s.emit_mode = self.EMIT.get(emit_mode, -1)
        s.ordered, s.sides, s.max_sessions_per_key = int(ordered), sides, max_sessions_per_key
        s.gap_us, s.wait_us = gap_us, N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_queued_rows, s.max_batch_rows = capacity_hint, max_queued_rows, max_batch_rows
        s.max_emit_rows, s.max_late_rows, s.max_product_rows = max_emit_rows, max_late_rows, max_product_rows
        self._create(ctx, s, sides)


@dataclass
class CollectWindowRows:
    """Rows of one ``CollectWindow.advance`` / ``eof``, each stream in the reference's downstream order, and the handles
    released since the previous one.  Each down row is a closed window: its list is
    ``handle[down_offset[i]:down_offset[i + 1]]`` in play order, and its metadata row follows it (``window_bounds``)."""

    down_key: np.ndarray
    down_window_id: np.ndarray
    down_epoch: np.ndarray
    down_offset: np.ndarray  # n_down + 1
    handle: np.ndarray
    late_key: np.ndarray
    late_window_id: np.ndarray
    late_epoch: np.ndarray
    late_activation: np.ndarray
    late_row: np.ndarray
    released: np.ndarray  # uint64, in no particular order

    def lists(self) -> List[List[int]]:
        """The handles of every down row, in play order."""
        h, o = self.handle.tolist(), self.down_offset.tolist()
        return [h[o[i]:o[i + 1]] for i in range(len(o) - 1)]


class CollectWindow:
    """``collect_window`` over tumbling or sliding windows (``bw_collect``, K9; windowing.py:1046-1190, 1436-1576).
    Values travel as uint64 handles; the caller keeps the objects, builds each window's container from its handles and
    may drop each object once its handle comes back in ``released``."""

    def __init__(self, ctx: Context, ordered: bool = True, length_us: int = 10_000_000, offset_us: Optional[int] = None,
                 align_us: int = 0, wait_us: Optional[int] = 0, capacity_hint: int = 1 << 16, max_windows_per_key: int = 16,
                 max_queued_rows: int = 1 << 20, max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20,
                 max_late_rows: int = 1 << 20):
        """``offset_us=None``: tumbling.  ``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``)."""
        self.ctx, self.lib = ctx, ctx.lib
        s = N.BwCollectSpec()
        s.struct_size = C.sizeof(N.BwCollectSpec)
        s.ordered, s.max_windows_per_key = int(ordered), max_windows_per_key
        s.length_us, s.offset_us, s.align_us = length_us, length_us if offset_us is None else offset_us, align_us
        s.wait_us = N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_queued_rows, s.max_batch_rows = capacity_hint, max_queued_rows, max_batch_rows
        s.max_emit_rows, s.max_late_rows = max_emit_rows, max_late_rows
        self.spec = s
        h = C.c_void_p()
        N.check(self.lib.bw_collect_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def window_bounds(self, window_id: int):
        """``(open_us, close_us)`` of a window (windowing.py:620-623)."""
        o = self.spec.align_us + self.spec.offset_us * window_id
        return o, o + self.spec.length_us

    def apply(self, keys, handles, ts_us, epoch: Optional[int] = None, system_now_us: int = 0):
        """One activation from host arrays.  ``system_now_us``: ``now_getter()`` of the activation."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        ts = np.ascontiguousarray(ts_us, dtype=np.int64)
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_collect_apply(self.h, vp(keys), vp(handles), vp(ts), keys.shape[0], epoch, int(system_now_us)), self.ctx.h)

    def apply_device(self, d_keys: int, d_handles: int, d_ts: int, rows: int, epoch: Optional[int] = None, system_now_us: int = 0):
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        N.check(self.lib.bw_collect_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_handles), C.c_void_p(d_ts), rows, epoch,
                                                 int(system_now_us)), self.ctx.h)

    def _wrap(self, r: N.BwCollectRows) -> CollectWindowRows:
        nd, nl, nr = int(r.n_down), int(r.n_late), int(r.n_released)

        def arr(ptr, n, dt=np.uint64):
            return np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).copy() if n else np.zeros(0, dt)

        off = arr(r.down_offset, nd + 1)
        return CollectWindowRows(arr(r.down_key, nd), arr(r.down_window_id, nd, np.int64), arr(r.down_epoch, nd), off,
                                 arr(r.handle, int(off[-1])), arr(r.late_key, nl), arr(r.late_window_id, nl, np.int64),
                                 arr(r.late_epoch, nl), arr(r.late_activation, nl), arr(r.late_row, nl), arr(r.released, nr))

    def advance(self, system_now_us: int = 0) -> CollectWindowRows:
        """Rows since the last call; ``system_now_us`` > 0 first runs the notify phase at that system time."""
        r = N.BwCollectRows()
        N.check(self.lib.bw_collect_advance(self.h, int(system_now_us), C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self) -> CollectWindowRows:
        r = N.BwCollectRows()
        N.check(self.lib.bw_collect_eof(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self.lib.bw_collect_destroy(self.h)
            self.h = None


@dataclass
class KeyCollectRows:
    """Lists of one ``KeyCollect.advance`` / ``eof``, in the reference's downstream order: per call, ascending key string,
    a key's lists in the order they filled.  List i is ``handle[offset[i]:offset[i + 1]]`` in arrival order; every
    handle passed to ``apply`` comes back exactly once, in the list that holds it."""

    key: np.ndarray
    epoch: np.ndarray
    offset: np.ndarray  # len(key) + 1
    handle: np.ndarray

    def lists(self) -> List[List[int]]:
        """The handles of every list, in arrival order."""
        h, o = self.handle.tolist(), self.offset.tolist()
        return [h[o[i]:o[i + 1]] for i in range(len(o) - 1)]


class KeyCollect:
    """The keyed ``collect(timeout, max_size)`` (``bw_kcollect``, K13; operators/__init__.py:1113-1216).  Values travel as
    uint64 handles; the caller keeps the objects and builds each list from its handles.  ``max_size`` must be >= 1."""

    def __init__(self, ctx: Context, max_size: int, capacity_hint: int = 1 << 16, max_batch_rows: int = 1 << 20,
                 max_emit_rows: int = 1 << 20):
        self.ctx, self.lib = ctx, ctx.lib
        s = N.BwKcollectSpec()
        s.struct_size = C.sizeof(N.BwKcollectSpec)
        s.max_size, s.capacity_hint, s.max_batch_rows, s.max_emit_rows = max_size, capacity_hint, max_batch_rows, max_emit_rows
        self.spec = s
        h = C.c_void_p()
        N.check(self.lib.bw_kcollect_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def _next_epoch(self, epoch: Optional[int]) -> int:
        if epoch is None:
            self._epoch += 1
            return self._epoch
        return epoch

    def apply(self, keys, handles, epoch: Optional[int] = None, timeout_at_us: int = 0):
        """One activation from host arrays.  ``timeout_at_us``: the activation's ``now_getter() + timeout``."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_kcollect_apply(self.h, vp(keys), vp(handles), keys.shape[0], self._next_epoch(epoch), int(timeout_at_us)),
                self.ctx.h)

    def apply_device(self, d_keys: int, d_handles: int, rows: int, epoch: Optional[int] = None, timeout_at_us: int = 0):
        N.check(self.lib.bw_kcollect_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_handles), rows, self._next_epoch(epoch),
                                                  int(timeout_at_us)), self.ctx.h)

    def _wrap(self, r: N.BwKcollectRows) -> KeyCollectRows:
        n = int(r.n)

        def arr(ptr, k):
            return np.ctypeslib.as_array(ptr, shape=(k,)).copy() if k else np.zeros(0, np.uint64)

        off = arr(r.offset, n + 1)
        return KeyCollectRows(arr(r.key, n), arr(r.epoch, n), off, arr(r.handle, int(off[-1])))

    def advance(self, now_us: int = 0) -> KeyCollectRows:
        """Lists since the last call; ``now_us`` > 0 first emits every list whose timeout is <= ``now_us``."""
        r = N.BwKcollectRows()
        N.check(self.lib.bw_kcollect_advance(self.h, int(now_us), C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self) -> KeyCollectRows:
        r = N.BwKcollectRows()
        N.check(self.lib.bw_kcollect_eof(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self.lib.bw_kcollect_destroy(self.h)
            self.h = None


@dataclass
class KeyJoinRows:
    """Rows of one ``KeyJoin.advance`` / ``eof`` in the reference's downstream order: per call, ascending key string, a
    key's emissions in item order, each emission's tuples in ``itertools.product`` order; and the handles released since
    the previous one."""

    key: np.ndarray
    handles: np.ndarray  # [rows, sides] uint64; valid where the side's bit of mask is set
    mask: np.ndarray
    epoch: np.ndarray
    released: np.ndarray  # uint64, in no particular order

    def tuples(self) -> List[tuple]:
        """The joined tuple of every row: a handle per side, None where the side's list was empty."""
        m = self.mask.tolist()
        return [tuple(int(h[s]) if mk >> s & 1 else None for s in range(len(h))) for h, mk in zip(self.handles.tolist(), m)]


class KeyJoin:
    """The keyed ``op.join`` with 1 to 4 sides and any insert mode (``bw_kjoin``, K15; ``_JoinLogic`` + ``_JoinState``,
    operators/__init__.py:2076-2190).  Each row is one tuple of an emission's ``itertools.product``, expanded on the
    device; values travel as uint64 handles, and each comes back in ``released`` once no list holds it."""

    INSERT = {"first": 0, "last": 1, "product": 2}
    EMIT = {"complete": 0, "final": 1, "running": 2}

    def __init__(self, ctx: Context, insert_mode: str = "product", emit_mode: str = "final", sides: int = 2, capacity_hint: int = 1 << 16,
                 max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20, max_product_rows: int = 1 << 26):
        """``max_product_rows``: rows one ``advance`` / ``eof`` may hand out."""
        self.ctx, self.lib, self.sides = ctx, ctx.lib, sides
        s = N.BwKjoinSpec()
        s.struct_size = C.sizeof(N.BwKjoinSpec)
        s.insert_mode, s.emit_mode, s.sides = self.INSERT.get(insert_mode, -1), self.EMIT.get(emit_mode, -1), sides
        s.capacity_hint, s.max_batch_rows, s.max_emit_rows, s.max_product_rows = capacity_hint, max_batch_rows, max_emit_rows, max_product_rows
        self.spec = s
        h = C.c_void_p()
        N.check(self.lib.bw_kjoin_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def _next_epoch(self, epoch: Optional[int]) -> int:
        if epoch is None:
            self._epoch += 1
            return self._epoch
        return epoch

    def apply(self, keys, sides, handles, epoch: Optional[int] = None):
        """One activation from host arrays: ``sides[i]`` is the side (0 .. sides-1) of item i."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        sides = np.ascontiguousarray(sides, dtype=np.uint8)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_kjoin_apply(self.h, vp(keys), vp(sides), vp(handles), keys.shape[0], self._next_epoch(epoch)), self.ctx.h)

    def apply_device(self, d_keys: int, d_sides: int, d_handles: int, rows: int, epoch: Optional[int] = None):
        N.check(self.lib.bw_kjoin_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_sides), C.c_void_p(d_handles), rows,
                                               self._next_epoch(epoch)), self.ctx.h)

    def _wrap(self, r: N.BwKjoinRows) -> KeyJoinRows:
        n, nr = int(r.n), int(r.n_released)

        def arr(ptr, k):
            return np.ctypeslib.as_array(ptr, shape=(k,)).copy() if k else np.zeros(0, np.uint64)

        hs = np.stack([arr(r.handle[s], n) for s in range(self.sides)], axis=1) if n else np.zeros((0, self.sides), np.uint64)
        return KeyJoinRows(arr(r.key, n), hs, arr(r.mask, n), arr(r.epoch, n), arr(r.released, nr))

    def advance(self) -> KeyJoinRows:
        """Rows since the last call."""
        r = N.BwKjoinRows()
        N.check(self.lib.bw_kjoin_advance(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self) -> KeyJoinRows:
        """End of input: "final" emits every key's product; every handle still held is released."""
        r = N.BwKjoinRows()
        N.check(self.lib.bw_kjoin_eof(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self.lib.bw_kjoin_destroy(self.h)
            self.h = None


@dataclass
class SessionCollectWindowRows(CollectWindowRows):
    """Rows of one ``SessionCollectWindow.advance`` / ``eof``.  Each down row is a closed session: its handles in
    flattened play order (``lists()``), its merge intervals (``merges(i)``) and its ``M`` row's bounds and merged ids
    (``merged(i)``).  Late rows all have window id -1 (``LATE_SESSION_ID``)."""

    open_us: np.ndarray = None
    close_us: np.ndarray = None
    merged_off: np.ndarray = None  # [n_down + 1] into merged_ids
    merged_ids: np.ndarray = None
    merge_off: np.ndarray = None  # [n_down + 1] into merge_start / merge_end
    merge_start: np.ndarray = None
    merge_end: np.ndarray = None

    def merged(self, i: int) -> List[int]:
        """The ids merged directly into down row ``i``'s session, ascending."""
        return self.merged_ids[self.merged_off[i] : self.merged_off[i + 1]].tolist()

    def merges(self, i: int) -> List[Tuple[int, int]]:
        """Down row ``i``'s merge intervals ``(start, end)`` into its list: each block one merged-away session's values,
        transitive merges included, by start ascending then end descending (the merge tree in pre-order)."""
        a, b = int(self.merge_off[i]), int(self.merge_off[i + 1])
        return list(zip(self.merge_start[a:b].tolist(), self.merge_end[a:b].tolist()))


class SessionCollectWindow:
    """``collect_window`` over session windows (``bw_scwin``, K12; windowing.py:671-810, 1046-1190, 1436-1576).  Values
    travel as uint64 handles; the caller keeps the objects, builds each session's container from its handles and merge
    intervals, and may drop each object once its handle comes back in ``released``."""

    def __init__(self, ctx: Context, ordered: bool = True, gap_us: int = 10_000_000, wait_us: Optional[int] = 0,
                 capacity_hint: int = 1 << 16, max_sessions_per_key: int = 16, max_queued_rows: int = 1 << 20,
                 max_batch_rows: int = 1 << 20, max_emit_rows: int = 1 << 20, max_late_rows: int = 1 << 20):
        """``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``)."""
        self.ctx, self.lib = ctx, ctx.lib
        s = N.BwScwinSpec()
        s.struct_size = C.sizeof(N.BwScwinSpec)
        s.ordered, s.max_sessions_per_key = int(ordered), max_sessions_per_key
        s.gap_us, s.wait_us = gap_us, N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_queued_rows, s.max_batch_rows = capacity_hint, max_queued_rows, max_batch_rows
        s.max_emit_rows, s.max_late_rows = max_emit_rows, max_late_rows
        self.spec = s
        h = C.c_void_p()
        N.check(self.lib.bw_scwin_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def _next_epoch(self, epoch: Optional[int]) -> int:
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        return epoch

    def apply(self, keys, handles, ts_us, epoch: Optional[int] = None, system_now_us: int = 0):
        """One activation from host arrays.  ``system_now_us``: ``now_getter()`` of the activation."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        ts = np.ascontiguousarray(ts_us, dtype=np.int64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_scwin_apply(self.h, vp(keys), vp(handles), vp(ts), keys.shape[0], self._next_epoch(epoch), int(system_now_us)),
                self.ctx.h)

    def apply_device(self, d_keys: int, d_handles: int, d_ts: int, rows: int, epoch: Optional[int] = None, system_now_us: int = 0):
        N.check(self.lib.bw_scwin_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_handles), C.c_void_p(d_ts), rows,
                                               self._next_epoch(epoch), int(system_now_us)), self.ctx.h)

    def _wrap(self, r: N.BwScwinRows) -> SessionCollectWindowRows:
        nd, nl, nr = int(r.n_down), int(r.n_late), int(r.n_released)

        def arr(ptr, n, dt=np.uint64):
            return np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).copy() if n else np.zeros(0, dt)

        off, moff, ioff = arr(r.down_offset, nd + 1), arr(r.merged_off, nd + 1), arr(r.merge_off, nd + 1)
        return SessionCollectWindowRows(arr(r.down_key, nd), arr(r.down_window_id, nd, np.int64), arr(r.down_epoch, nd), off,
                                        arr(r.handle, int(off[-1])), arr(r.late_key, nl), np.full(nl, -1, np.int64),
                                        arr(r.late_epoch, nl), arr(r.late_activation, nl), arr(r.late_row, nl), arr(r.released, nr),
                                        arr(r.open_us, nd, np.int64), arr(r.close_us, nd, np.int64), moff,
                                        arr(r.merged_ids, int(moff[-1]), np.int64), ioff, arr(r.merge_start, int(ioff[-1])),
                                        arr(r.merge_end, int(ioff[-1])))

    def advance(self, system_now_us: int = 0) -> SessionCollectWindowRows:
        """Rows since the last call; ``system_now_us`` > 0 first runs the notify phase at that system time."""
        r = N.BwScwinRows()
        N.check(self.lib.bw_scwin_advance(self.h, int(system_now_us), C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self) -> SessionCollectWindowRows:
        r = N.BwScwinRows()
        N.check(self.lib.bw_scwin_eof(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self.lib.bw_scwin_destroy(self.h)
            self.h = None


@dataclass
class ArgWindowRows:
    """Rows of one ``ArgWindow.advance`` / ``eof``, each stream in the reference's downstream order, and the handles
    released since the previous one.  Each closed row is a window's ``E`` row (the pick's handle) followed by its ``M``
    row ``WindowMetadata(open, close[, merged ids])``.  Session late rows have window id -1 (``LATE_SESSION_ID``)."""

    closed_key: np.ndarray
    closed_window_id: np.ndarray
    closed_handle: np.ndarray
    closed_open_us: np.ndarray
    closed_close_us: np.ndarray
    closed_epoch: np.ndarray
    merged_off: np.ndarray  # [n_closed + 1] into merged_ids
    merged_ids: np.ndarray
    late_key: np.ndarray
    late_window_id: np.ndarray
    late_epoch: np.ndarray
    late_activation: np.ndarray
    late_row: np.ndarray
    released: np.ndarray  # uint64, in no particular order

    def merged(self, i: int) -> List[int]:
        """The ids merged directly into closed row ``i``'s session, ascending (none for tumbling / sliding windows)."""
        return self.merged_ids[self.merged_off[i] : self.merged_off[i + 1]].tolist()


class ArgWindow:
    """``max_window`` / ``min_window`` with a ``by=`` projection over tumbling, sliding or session windows (``bw_argwin``,
    K11; windowing.py:1046-1190, 1692-1714, 2145-2285).  Items travel as uint64 handles with their by-values (int64 or
    float64); the caller keeps the items and may drop each one once its handle comes back in ``released``."""

    EXTREME = {"max": N.RED["max"], "min": N.RED["min"]}

    def __init__(self, ctx: Context, extreme: str = "max", by_dtype: str = "i64", length_us: int = 10_000_000,
                 offset_us: Optional[int] = None, align_us: int = 0, gap_us: Optional[int] = None, wait_us: Optional[int] = 0,
                 capacity_hint: int = 1 << 16, max_windows_per_key: int = 16, max_batch_rows: int = 1 << 20,
                 max_emit_rows: int = 1 << 20, max_late_rows: int = 1 << 20):
        """``gap_us`` set: session windows (``length_us`` / ``offset_us`` / ``align_us`` unused).  ``offset_us=None``:
        tumbling.  ``wait_us=None``: the watermark never advances on data (``BW_WAIT_FOREVER``)."""
        self.ctx, self.lib = ctx, ctx.lib
        self.by_dtype = by_dtype
        s = N.BwArgwinSpec()
        s.struct_size = C.sizeof(N.BwArgwinSpec)
        s.extreme, s.by_dtype = self.EXTREME.get(extreme, -1), N.VAL.get(by_dtype, -1)
        s.session, s.max_windows_per_key = int(gap_us is not None), max_windows_per_key
        s.length_us, s.offset_us, s.align_us = length_us, length_us if offset_us is None else offset_us, align_us
        s.gap_us = 0 if gap_us is None else gap_us
        s.wait_us = N.BW_WAIT_FOREVER if wait_us is None else wait_us
        s.capacity_hint, s.max_batch_rows, s.max_emit_rows, s.max_late_rows = capacity_hint, max_batch_rows, max_emit_rows, max_late_rows
        self.spec = s
        h = C.c_void_p()
        N.check(self.lib.bw_argwin_create(ctx.h, C.byref(s), C.byref(h)), ctx.h)
        self.h = h
        self._epoch = 0

    def _next_epoch(self, epoch: Optional[int]) -> int:
        if epoch is None:
            self._epoch += 1
            epoch = self._epoch
        return epoch

    def apply(self, keys, handles, by, ts_us, epoch: Optional[int] = None, system_now_us: int = 0):
        """One activation from host arrays; ``by`` holds the by-values (int64 or float64 as the step's ``by_dtype``).
        ``system_now_us``: ``now_getter()`` of the activation."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        b = np.ascontiguousarray(by, dtype=np.float64 if self.by_dtype == "f64" else np.int64)
        ts = np.ascontiguousarray(ts_us, dtype=np.int64)
        epoch = self._next_epoch(epoch)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        N.check(self.lib.bw_argwin_apply(self.h, vp(keys), vp(handles), vp(b), vp(ts), keys.shape[0], epoch, int(system_now_us)), self.ctx.h)

    def apply_device(self, d_keys: int, d_handles: int, d_by: int, d_ts: int, rows: int, epoch: Optional[int] = None,
                     system_now_us: int = 0):
        epoch = self._next_epoch(epoch)
        N.check(self.lib.bw_argwin_apply_device(self.h, C.c_void_p(d_keys), C.c_void_p(d_handles), C.c_void_p(d_by), C.c_void_p(d_ts),
                                                rows, epoch, int(system_now_us)), self.ctx.h)

    def _wrap(self, r: N.BwArgwinRows) -> ArgWindowRows:
        nc, nl, nr = int(r.n_closed), int(r.n_late), int(r.n_released)

        def arr(ptr, n, dt=np.uint64):
            return np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).copy() if n else np.zeros(0, dt)

        off = arr(r.merged_off, nc + 1).astype(np.int64)
        return ArgWindowRows(arr(r.closed_key, nc), arr(r.closed_window_id, nc, np.int64), arr(r.closed_handle, nc),
                             arr(r.closed_open_us, nc, np.int64), arr(r.closed_close_us, nc, np.int64), arr(r.closed_epoch, nc), off,
                             arr(r.merged_ids, int(off[-1]), np.int64), arr(r.late_key, nl), arr(r.late_window_id, nl, np.int64),
                             arr(r.late_epoch, nl), arr(r.late_activation, nl), arr(r.late_row, nl), arr(r.released, nr))

    def advance(self, system_now_us: int = 0) -> ArgWindowRows:
        """Rows since the last call; ``system_now_us`` > 0 first runs the notify phase at that system time."""
        r = N.BwArgwinRows()
        N.check(self.lib.bw_argwin_advance(self.h, int(system_now_us), C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def eof(self) -> ArgWindowRows:
        r = N.BwArgwinRows()
        N.check(self.lib.bw_argwin_eof(self.h, C.byref(r)), self.ctx.h)
        return self._wrap(r)

    def close(self):
        if self.h:
            self.lib.bw_argwin_destroy(self.h)
            self.h = None
