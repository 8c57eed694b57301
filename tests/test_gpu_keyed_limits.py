"""K7 - K11 at M = 32, 33, 63 and 64 sessions or windows per key (64: the engine's default) against their oracles.  -m gpu.

Every stream comes from tests/keyed_limits_streams.py, and what the device must do comes from the instrumented oracle
run: where no key of a call needs more than M records, merged ids or open windows, the device's rows (in its own order,
f64 by bits), merged ids and released handles equal the oracle's; at the first call that needs more, the call fails
with BW_ERR_CAPACITY and the kernel's own reason, after every earlier call matched, and the object refuses further
calls.  A cross-kernel check pins K7's inline session walk to the shared steps K10 and K11 call."""

import operator
import random
import struct
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

from bytewax_b200 import _native as N
from tests import keyed_limits_streams as ks
from tests.test_gpu_arg_window import _rows as aw_rows
from tests.test_gpu_collect_window import _rows as cw_rows
from tests.test_gpu_join_window import _rows as jw_rows
from tests.test_gpu_session_join import _rows as sj_rows
from tests.test_gpu_sessions import _rows as k7_rows
from tests.test_gpu_sessions import _same

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = ks.S, ks.A
SMALL = dict(capacity_hint=1 << 10, max_batch_rows=1 << 16, max_emit_rows=1 << 18, max_late_rows=1 << 16)


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _wait(spec):
    return None if spec["wait_us"] == ks.WAIT_FOREVER else spec["wait_us"]


def _wrap_i64(x):
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def _play(obj, steps, feed, fail_at, reason):
    """Feed steps then EOF; ``fail_at``: the step (``len(steps)``: EOF) that must fail with ``reason``.  Returns the
    converted output of every step before it."""
    got = []
    try:
        for i, step in enumerate(list(steps) + [None]):
            if i == fail_at:
                with pytest.raises(N.BwError) as ei:
                    feed(obj, step, i)
                assert ei.value.status == 3 and reason in str(ei.value), str(ei.value)
                with pytest.raises(N.BwError) as ei:
                    obj.advance()
                assert ei.value.status == 5
                return got
            got.append(feed(obj, step, i))
    finally:
        obj.close()
    assert fail_at is None
    return got


# ---------------------------------------------------------------------------
# K7
# ---------------------------------------------------------------------------


def _k7_run(ctx, spec, steps, M):
    from bytewax_b200 import gpu

    f = gpu.SessionFold(ctx, spec["reduction"], spec["gap_us"], _wait(spec), val_dtype=spec["val_dtype"], max_sessions_per_key=M, **SMALL)
    dt = np.float64 if spec["val_dtype"] == "f64" else np.int64
    n_act = [0]

    def feed(f, step, i):
        if step is None:
            return k7_rows(f.eof(), None)
        if step[0] == "notify":
            return k7_rows(f.advance(system_now_us=step[1]), None)
        _, now, keys, ts, vals = step
        f.apply(np.array(keys, np.uint64), None if spec["reduction"] == "count" else np.array(vals, dtype=dt), np.array(ts, np.int64),
                epoch=i + 1, system_now_us=now)
        out = k7_rows(f.advance(), (n_act[0], vals))
        n_act[0] += 1
        return out

    return f, feed


def _k7_want(spec, steps):
    acts, logs = ks.measure("k7", spec, steps)
    if spec["reduction"] == "sum" and spec["val_dtype"] == "i64":  # the device's i64 sums wrap past 2^63
        acts = [[[k, w, t, _wrap_i64(p) if t == "E" else p] for k, w, t, p in a] for a in acts]
    return acts, logs


K7_FOLDS = [("sum", "f64"), ("sum", "i64"), ("max", "f64"), ("min", "f64"), ("count", "i64")]


def _variants(M, all_of):
    """Every variant at M = 63 / 64, where the high mask bits and indices are reached; the first two below that, where
    only the counts' bounds are (this keeps the file's time near two minutes)."""
    return all_of if M >= 63 else all_of[:2]


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_k7_session_builders(ctx, M, builder):
    clock, steps0 = ks.session_builders(M)[builder]
    for red, dtype in _variants(M, K7_FOLDS):
        spec, steps = ks.for_kernel("k7", clock, steps0 if dtype == "f64" else ks.revalue(steps0, "i64", M), reduction=red, val_dtype=dtype)
        want, logs = _k7_want(spec, steps)
        fail = ks.first_overflow(logs, M)
        f, feed = _k7_run(ctx, spec, steps, M)
        got = _play(f, steps, feed, fail, "max_sessions_per_key sessions or merged ids")
        assert _same(got, want[: len(got)]), (red, dtype)


# ---------------------------------------------------------------------------
# K10 and K11 sessions
# ---------------------------------------------------------------------------


def _feeder(rows_of, extra):
    """feed() for a handle kernel: ``extra`` applies a batch step; returns (rows, sorted released handles) per step."""
    n_act = [0]

    def feed(o, step, i):
        if step is None:
            out = o.eof()
            batch = None
        elif step[0] == "notify":
            out = o.advance(system_now_us=step[1])
            batch = None
        else:
            extra(o, step, i)
            out = o.advance()
            batch = step
        r = rows_of(out, batch, n_act[0])
        if batch is not None:
            n_act[0] += 1
        return r, sorted(out.released.tolist())

    return feed


def _k10(ctx, clock, steps0, M, ordered, sides, mode):
    from bytewax_b200 import gpu

    ins, emit = mode
    spec, steps = ks.for_kernel("k10", clock, steps0, insert_mode=ins, emit_mode=emit, ordered=ordered, sides=sides)
    (want, want_rel), logs = ks.measure("k10", spec, steps)
    fail = ks.first_overflow(logs, M)
    j = gpu.SessionJoinWindow(ctx, ins, emit, ordered, sides, spec["gap_us"], _wait(spec), max_sessions_per_key=M,
                              max_queued_rows=1 << 16, **SMALL)

    def apply(o, step, i):
        _, now, keys, ts, sd, hs = step
        o.apply(np.array(keys, np.uint64), np.array(sd, np.uint8), np.array(hs, np.uint64), np.array(ts, np.int64), epoch=i + 1,
                system_now_us=now)

    rows = lambda out, b, act: sj_rows(out, None if b is None else dict(act=act, sides=b[4], vals=b[5]), emit == "final")  # noqa: E731
    got = _play(j, steps, _feeder(rows, apply), fail, "max_sessions_per_key sessions or merged ids")
    assert [g[0] for g in got] == want[: len(got)]
    assert [g[1] for g in got] == want_rel[: len(got)]
    return got, want, fail


K10_CASES = [(False, 1, ("first", "final")), (True, 1, ("last", "running")), (False, 4, ("last", "complete")), (True, 4, ("first", "final"))]


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_k10_session_builders(ctx, M, builder):
    clock, steps0 = ks.session_builders(M)[builder]
    for ordered, sides, mode in _variants(M, K10_CASES):
        got, want, fail = _k10(ctx, clock, steps0, M, ordered, sides, mode)
        if fail is None:  # every handle released exactly once
            flat = [h for g in got for h in g[1]]
            assert sorted(flat) == list(range(sum(len(s[2]) for s in steps0 if s[0] == "batch")))


def _k11(ctx, clock, steps0, M, extreme, f64=True):
    from bytewax_b200 import gpu

    spec, steps = ks.for_kernel("k11", clock, steps0, extreme=extreme)
    (want, want_rel), logs = ks.measure("k11", spec, steps)
    fail = ks.first_overflow(logs, M)
    session = "gap_us" in spec
    if session:
        a = gpu.ArgWindow(ctx, extreme, "f64" if f64 else "i64", gap_us=spec["gap_us"], wait_us=_wait(spec), max_windows_per_key=M, **SMALL)
    else:
        a = gpu.ArgWindow(ctx, extreme, "f64" if f64 else "i64", spec["length_us"], spec["offset_us"], spec["align_us"], wait_us=_wait(spec),
                          max_windows_per_key=M, **SMALL)

    def apply(o, step, i):
        _, now, keys, ts, bys, hs = step
        o.apply(np.array(keys, np.uint64), np.array(hs, np.uint64), np.array([ks.aw.dec(b) for b in bys], np.float64 if f64 else np.int64),
                np.array(ts, np.int64), epoch=i + 1, system_now_us=now)

    rows = lambda out, b, act: aw_rows(out, None if b is None else dict(act=act, handles=b[5]), session)  # noqa: E731
    reason = "max_windows_per_key sessions or merged ids" if session else "max_windows_per_key open windows"
    got = _play(a, steps, _feeder(rows, apply), fail, reason)
    assert [g[0] for g in got] == want[: len(got)]
    assert [g[1] for g in got] == want_rel[: len(got)]
    if fail is None:
        flat = [h for g in got for h in g[1]]
        assert sorted(flat) == list(range(sum(len(s[2]) for s in steps0 if s[0] == "batch")))
    return got


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_k11_session_builders(ctx, M, builder):
    clock, steps0 = ks.session_builders(M)[builder]
    for extreme in ("max", "min"):
        _k11(ctx, clock, steps0, M, extreme)


# ---------------------------------------------------------------------------
# the same stream through K7, K10 and K11: K7's inline walk against the shared steps
# ---------------------------------------------------------------------------


def _bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _sessions_of(rows):
    """Per call: the M rows (key, id, [open, close, merged]) and the late rows' keys, in the device's order."""
    return [([(r[0], r[1], r[3]) for r in a if r[2] == "M"], [r[0] for r in a if r[2] == "L"]) for a in rows]


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_cross_kernel_sessions(ctx, M, builder):
    clock, steps0 = ks.session_builders(M)[builder]
    k7 = {}
    for red in ("count", "sum", "max", "min"):
        spec, steps = ks.for_kernel("k7", clock, steps0, reduction=red, val_dtype="f64")
        fail = ks.first_overflow(ks.measure("k7", spec, steps)[1], M)
        f, feed = _k7_run(ctx, spec, steps, M)
        k7[red] = (_play(f, steps, feed, fail, "max_sessions_per_key"), fail)
    fails = {fail for _, fail in k7.values()}
    assert len(fails) == 1
    shape = _sessions_of(k7["count"][0])
    for red in ("sum", "max", "min"):
        assert _sessions_of(k7[red][0]) == shape, red
    k10, _, fail10 = _k10(ctx, clock, steps0, M, False, 1, ("first", "final"))
    assert {fail10} == fails
    assert _sessions_of([g[0] for g in k10]) == shape
    by = {}
    nxt = 0
    for s in steps0:
        if s[0] == "batch":
            for v in s[4]:
                by[nxt] = v
                nxt += 1
    for extreme in ("max", "min"):
        got = _k11(ctx, clock, steps0, M, extreme)
        rows = [g[0] for g in got]
        assert _sessions_of(rows) == shape, extreme
        picks = [by[r[3]] for a in rows for r in a if r[2] == "E"]
        accs = [r[3] for a in k7[extreme][0] for r in a if r[2] == "E"]
        assert [_bits(x) for x in picks] == [_bits(x) for x in accs], extreme  # signed zeros and NaN included


# ---------------------------------------------------------------------------
# K8, K9 and K11 over tumbling and sliding windows
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.WINDOW_BUILDERS)
def test_k9_window_builders(ctx, M, builder):
    from bytewax_b200 import gpu

    clock, steps0 = ks.window_builders(M)[builder]
    for ordered in (False, True):
        spec, steps = ks.for_kernel("k9", clock, steps0, ordered=ordered)
        (want, want_rel), logs = ks.measure("k9", spec, steps)
        fail = ks.first_overflow(logs, M)
        c = gpu.CollectWindow(ctx, ordered, spec["length_us"], spec["offset_us"], spec["align_us"], _wait(spec), max_windows_per_key=M,
                              max_queued_rows=1 << 16, **SMALL)

        def apply(o, step, i):
            _, now, keys, ts, _sd, hs = step
            o.apply(np.array(keys, np.uint64), np.array(hs, np.uint64), np.array(ts, np.int64), epoch=i + 1, system_now_us=now)

        rows = lambda out, b, act: cw_rows(out, c.window_bounds, dict(act=act, vals=b[5]) if b is not None else dict(act=None))  # noqa: E731
        got = _play(c, steps, _feeder(rows, apply), fail, "max_windows_per_key open windows")
        assert [g[0] for g in got] == want[: len(got)], ordered
        assert [g[1] for g in got] == want_rel[: len(got)], ordered


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.WINDOW_BUILDERS)
def test_k8_window_builders(ctx, M, builder):
    from bytewax_b200 import gpu

    clock, steps0 = ks.window_builders(M)[builder]
    for k, (ins, emit) in enumerate(_variants(M, ks.jo.MODES)):
        ordered = k % 2 == 0  # (each mode in one of ordered / unordered, alternating: both queues, every mode)
        spec, steps = ks.for_kernel("k8", clock, steps0, insert_mode=ins, emit_mode=emit, ordered=ordered, sides=4)
        (want, want_rel), logs = ks.measure("k8", spec, steps)
        fail = ks.first_overflow(logs, M)
        j = gpu.JoinWindow(ctx, ins, emit, ordered, 4, spec["length_us"], spec["offset_us"], spec["align_us"], _wait(spec),
                           max_windows_per_key=M, max_queued_rows=1 << 16, **SMALL)

        def apply(o, step, i):
            _, now, keys, ts, sd, hs = step
            o.apply(np.array(keys, np.uint64), np.array(sd, np.uint8), np.array(hs, np.uint64), np.array(ts, np.int64), epoch=i + 1,
                    system_now_us=now)

        final = emit == "final"
        rows = lambda out, b, act: jw_rows(out, j.window_bounds, dict(act=act, sides=b[4], vals=b[5], final=final) if b is not None  # noqa: E731
                                           else dict(act=None, final=final))
        got = _play(j, steps, _feeder(rows, apply), fail, "max_windows_per_key open windows")
        assert [g[0] for g in got] == want[: len(got)], (ins, emit)
        assert [g[1] for g in got] == want_rel[: len(got)], (ins, emit)


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.WINDOW_BUILDERS)
def test_k11_window_builders(ctx, M, builder):
    clock, steps0 = ks.window_builders(M)[builder]
    for extreme in ("max", "min"):
        _k11(ctx, clock, steps0, M, extreme, f64=False)


# ---------------------------------------------------------------------------
# engine: run_main(gpu=True) with a key of 64 sessions or windows, at the engine's default per-key limit
# ---------------------------------------------------------------------------


@pytest.fixture
def device_calls(monkeypatch):
    """Small key tables and batches (each keyed step would otherwise reserve GiBs), the per-key limit left at its
    default; records (class, per-key limit, rows) of every device activation."""
    from bytewax_b200 import gpu

    monkeypatch.setenv("BYTEWAX_B200_KEYS", "256")
    monkeypatch.setenv("BYTEWAX_B200_BATCH", "4096")
    monkeypatch.delenv("BYTEWAX_B200_SESSIONS", raising=False)
    calls = []
    for cls in (gpu.SessionFold, gpu.SessionJoinWindow, gpu.CollectWindow, gpu.ArgWindow):
        orig = cls.apply

        def apply(self, *a, _orig=orig, **k):
            s = self.spec
            calls.append((type(self).__name__, getattr(s, "max_sessions_per_key", None) or s.max_windows_per_key, len(a[0])))
            return _orig(self, *a, **k)

        monkeypatch.setattr(cls, "apply", apply)
    return calls


ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = ALIGN + timedelta(days=400)  # now_getter: the watermark moves on data only
ENGINE_F64 = ks.so.F64_VALUES + (0.0, -0.0)


def _engine_items(seed, windows):
    """A hot key with 64 sessions (2 s apart, gap 1 s) or 64 tumbling windows (10 s), opened in one activation in a
    seeded order, next to 8 light keys; sessions then get bridges (1 s after a session) that merge 40 of them, most at
    record indices >= 32.  Returns the two phases' items as (key, ts, i)."""
    rnd = random.Random(seed)
    step = 10 if windows else 2
    slots = list(range(64))
    rnd.shuffle(slots)
    first = [("hot", ALIGN + timedelta(seconds=step * p + (rnd.random() * 5 if windows else 0))) for p in slots for _ in range(rnd.randint(1, 2))]
    first += [(f"k{rnd.randrange(8)}", ALIGN + timedelta(seconds=rnd.uniform(0, 120))) for _ in range(60)]
    rnd.shuffle(first)
    second = [] if windows else [("hot", ALIGN + timedelta(seconds=2 * p + 1)) for p in rnd.sample(range(63), 40)]
    second += [(f"k{rnd.randrange(8)}", ALIGN + timedelta(seconds=rnd.uniform(0, 120))) for _ in range(len(first) - len(second))]
    return [(k, t, i) for i, (k, t) in enumerate(first + second)], len(first)


def _engine_both(build):
    from bytewax_b200.testing import run_main

    outs = []
    for on_gpu in (False, True):
        flow, sinks = build()
        run_main(flow, gpu=on_gpu)
        outs.append(sinks)
    return outs


def _engine_flow(streams_of, make, batch):
    import bytewax_b200.operators as op
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource

    down, late, meta = [], [], []
    flow = Dataflow("df")
    wo = make([op.input(f"in{i}", flow, TestingSource(items, batch_size=batch)) for i, items in enumerate(streams_of)])
    op.output("out", wo.down, TestingSink(down))
    op.output("late", wo.late, TestingSink(late))
    op.output("meta", wo.meta, TestingSink(meta))
    return flow, (down, late, meta)


def _hot(meta):
    """The hot key's closed sessions / windows, and the highest id among them and their merged ids."""
    rows = [(w, m) for k, (w, m) in meta if k == "hot"]
    return len(rows), max(max([w] + list(getattr(m, "merged_ids", ()) or ())) for w, m in rows)


class _F(float):
    pass


def _val(v, ts):
    x = _F(v)
    x.ts = ts
    return x


def test_engine_session_fold_64(device_calls):
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, SessionWindower

    items, n1 = _engine_items(1, False)
    rnd = random.Random(2)
    vals = [(k, _val(rnd.choice(ENGINE_F64), t)) for k, t, _ in items]

    def build():
        clock = EventClock(lambda v: v.ts, timedelta(days=1), now_getter=lambda: FROZEN)
        return _engine_flow([vals], lambda s: win.reduce_window("r", s[0], clock, SessionWindower(timedelta(seconds=1)), operator.add), n1)

    host, dev = _engine_both(build)
    bits = lambda rows: [(k, w, _bits(float(v))) for k, (w, v) in rows]  # noqa: E731
    assert bits(dev[0]) == bits(host[0]) and dev[1:] == host[1:]
    assert _hot(host[2])[0] == 24  # 64 sessions held at once (nothing closes before EOF), 40 bridges each merging two
    assert device_calls and all(c[:2] == ("SessionFold", 64) for c in device_calls) and device_calls[0][2] == n1


def test_engine_session_join_64(device_calls):
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, SessionWindower

    items, n1 = _engine_items(3, False)
    sides = [[(k, {"ts": t, "i": i}) for k, t, i in items if i % 2 == s] for s in (0, 1)]

    def build():
        clock = EventClock(lambda v: v["ts"], timedelta(days=1), now_getter=lambda: FROZEN)
        return _engine_flow(sides, lambda s: win.join_window("j", clock, SessionWindower(timedelta(seconds=1)), *s, insert_mode="first",
                                                             emit_mode="final", ordered=False), n1 // 2)

    host, dev = _engine_both(build)
    assert dev == host
    assert _hot(host[2])[0] == 24
    assert device_calls and all(c[:2] == ("SessionJoinWindow", 64) for c in device_calls)


def test_engine_collect_64(device_calls):
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, TumblingWindower

    items, n1 = _engine_items(4, True)

    def build():
        clock = EventClock(lambda v: v[0], timedelta(days=1), now_getter=lambda: FROZEN)
        return _engine_flow([[(k, (t, i)) for k, t, i in items]],
                            lambda s: win.collect_window("c", s[0], clock, TumblingWindower(timedelta(seconds=10), ALIGN), ordered=False), n1)

    host, dev = _engine_both(build)
    assert dev == host
    assert _hot(host[2]) == (64, 63)  # 64 windows open until EOF
    assert device_calls and all(c[:2] == ("CollectWindow", 64) for c in device_calls)


@pytest.mark.parametrize("windows", [False, True])
def test_engine_arg_window_64(device_calls, windows):
    import bytewax_b200.operators as op
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, SessionWindower, TumblingWindower

    items, n1 = _engine_items(5 + windows, windows)
    rnd = random.Random(7)
    recs = [{"user": k, "ts": t, "val": rnd.choice((-0.0, 0.0, 1.5, -2.0, float("inf"), float("nan")))} for k, t, _ in items]
    windower = TumblingWindower(timedelta(seconds=10), ALIGN) if windows else SessionWindower(timedelta(seconds=1))

    def build():
        clock = EventClock(lambda e: e["ts"], timedelta(days=1), now_getter=lambda: FROZEN)
        return _engine_flow([recs], lambda s: win.max_window("m", op.key_on("key", s[0], lambda e: e["user"]), clock, windower,
                                                             by=lambda e: e["val"]), n1)

    host, dev = _engine_both(build)
    assert dev == host  # (the same item objects in both runs: NaN by-values compare by identity)
    assert _hot(host[2]) == (64, 63) if windows else _hot(host[2])[0] == 24
    assert device_calls and all(c[:2] == ("ArgWindow", 64) for c in device_calls)
