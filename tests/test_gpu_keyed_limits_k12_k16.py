"""K12, K14 and K16 at M = 32, 33, 63 and 64 sessions or windows per key (64: the engine's default) against their
oracles.  -m gpu.

K12 (session ``collect_window``), K14 (product ``join_window`` over tumbling and sliding windows) and K16 (product
``join_window`` over sessions) keep a key's state as K7 - K11 do, in a fixed array of M records walked by one thread
with 64-bit cell masks, and this file drives them as tests/test_gpu_keyed_limits.py drives those: every stream comes
from tests/keyed_limits_streams.py, and what the device must do comes from the instrumented oracle run.  Where no key of
a call needs more than M records, merged ids, open windows or (K12) merge intervals, the device's rows equal the
oracle's call by call -- K12's lists in flattened play order with their merge intervals, K14's and K16's product rows
in ``itertools.product`` order -- and so do the handles each call releases; at the first call that needs more, the call
fails with BW_ERR_CAPACITY and the kernel's own reason, after every earlier call matched, and the object refuses
further calls.  A cross-kernel check pins K12's and K16's session walks to K10's, and three engine runs take each
kernel to 64 at the engine's default limit."""

import random
from datetime import timedelta

import numpy as np
import pytest

from tests import keyed_limits_streams as ks
from tests.test_gpu_keyed_limits import ALIGN, FROZEN, _engine_both, _engine_flow, _engine_items, _feeder, _hot, _k10, _play, _sessions_of, \
    _variants, _wait, SMALL
from tests.test_gpu_product_join_window import _rows as pj_rows
from tests.test_gpu_session_collect import _device_rows as sc_rows
from tests.test_gpu_session_product_join import _rows as sp_rows

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

K12_REASON = "max_sessions_per_key sessions, merged ids or merge intervals"
K14_REASON = "max_windows_per_key open windows"
K16_REASON = "max_sessions_per_key sessions or merged ids"


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _n_handles(steps0):
    return sum(len(s[2]) for s in steps0 if s[0] == "batch")


def _released_once(got, steps0):
    flat = [h for g in got for h in g[1]]
    assert sorted(flat) == list(range(_n_handles(steps0))), "a handle released twice or never"


# ---------------------------------------------------------------------------
# K12: collect_window over sessions
# ---------------------------------------------------------------------------


def _k12(ctx, clock, steps0, M, ordered):
    """The device against the instrumented oracle; per call before the failing one (if any): ((E, M, L rows), released)."""
    from bytewax_b200 import gpu

    spec, steps = ks.for_kernel("k12", clock, steps0, ordered=ordered)
    (want, want_rel), logs = ks.measure("k12", spec, steps)
    fail = ks.first_overflow(logs, M, "k12")
    c = gpu.SessionCollectWindow(ctx, ordered, spec["gap_us"], _wait(spec), max_sessions_per_key=M, max_queued_rows=1 << 16, **SMALL)

    def feed(o, step, i):
        if step is None:
            out, hs = o.eof(), []
        elif step[0] == "notify":
            out, hs = o.advance(system_now_us=step[1]), []
        else:
            _, now, keys, ts, hs = step
            o.apply(np.array(keys, np.uint64), np.array(hs, np.uint64), np.array(ts, np.int64), epoch=i + 1, system_now_us=now)
            out = o.advance()
        E, Mr, L, rel = sc_rows(out, hs)
        return (E, Mr, L), rel

    got = _play(c, steps, feed, fail, K12_REASON)
    split = [tuple([r for r in a if r[2] == tag] for tag in "EML") for a in want]
    assert [g[0] for g in got] == split[: len(got)], ordered
    assert [g[1] for g in got] == want_rel[: len(got)], ordered
    if fail is None:
        _released_once(got, steps0)
    return got, fail


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_k12_session_builders(ctx, M, builder):
    clock, steps0 = ks.session_builders(M)[builder]
    for ordered in (False, True):
        _k12(ctx, clock, steps0, M, ordered)


# ---------------------------------------------------------------------------
# K14: product join_window over tumbling and sliding windows
# ---------------------------------------------------------------------------


def _k14(ctx, clock, steps0, M, emit, sides, ordered):
    from bytewax_b200 import gpu

    spec, steps = ks.for_kernel("k14", clock, steps0, emit_mode=emit, ordered=ordered, sides=sides)
    (want, want_rel), logs = ks.measure("k14", spec, steps)
    fail = ks.first_overflow(logs, M)
    j = gpu.ProductJoinWindow(ctx, emit, ordered, sides, spec["length_us"], spec["offset_us"], spec["align_us"], _wait(spec),
                              max_windows_per_key=M, max_queued_rows=1 << 16, **SMALL)

    def apply(o, step, i):
        _, now, keys, ts, sd, hs = step
        o.apply(np.array(keys, np.uint64), np.array(sd, np.uint8), np.array(hs, np.uint64), np.array(ts, np.int64), epoch=i + 1,
                system_now_us=now)

    final = emit == "final"
    rows = lambda out, b, act: pj_rows(out, j.window_bounds, None if b is None else dict(sides=b[4], vals=b[5]), final)  # noqa: E731
    got = _play(j, steps, _feeder(rows, apply), fail, K14_REASON)
    assert [g[0] for g in got] == want[: len(got)], (emit, sides, ordered)
    assert [g[1] for g in got] == want_rel[: len(got)], (emit, sides, ordered)
    if fail is None:
        _released_once(got, steps0)
    return got


# every emit mode with every side count, ordered and not; the first two (all that runs below M = 63) differ in each
K14_CASES = [("complete", 2, False), ("running", 3, True)]
K14_CASES += [(e, s, o) for e in ks.po.EMITS for s in (1, 2, 3, 4) for o in (False, True) if (e, s, o) not in K14_CASES]


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.WINDOW_BUILDERS)
def test_k14_window_builders(ctx, M, builder):
    clock, steps0 = ks.window_builders(M)[builder]
    for emit, sides, ordered in _variants(M, K14_CASES):
        _k14(ctx, clock, steps0, M, emit, sides, ordered)


# ---------------------------------------------------------------------------
# K16: product join_window over sessions
# ---------------------------------------------------------------------------


def _k16(ctx, clock, steps0, M, emit, sides, ordered=False):
    from bytewax_b200 import gpu

    spec, steps = ks.for_kernel("k16", clock, steps0, emit_mode=emit, ordered=ordered, sides=sides)
    (want, want_rel), logs = ks.measure("k16", spec, steps)
    fail = ks.first_overflow(logs, M)
    j = gpu.SessionProductJoinWindow(ctx, emit, ordered, sides, spec["gap_us"], _wait(spec), max_sessions_per_key=M,
                                     max_queued_rows=1 << 16, **SMALL)

    def apply(o, step, i):
        _, now, keys, ts, sd, hs = step
        o.apply(np.array(keys, np.uint64), np.array(sd, np.uint8), np.array(hs, np.uint64), np.array(ts, np.int64), epoch=i + 1,
                system_now_us=now)

    final = emit == "final"
    rows = lambda out, b, act: sp_rows(out, None if b is None else dict(act=act, sides=b[4], vals=b[5]), final)  # noqa: E731
    got = _play(j, steps, _feeder(rows, apply), fail, K16_REASON)
    assert [g[0] for g in got] == want[: len(got)], (emit, sides, ordered)
    assert [g[1] for g in got] == want_rel[: len(got)], (emit, sides, ordered)
    if fail is None:
        _released_once(got, steps0)
    return got, fail


# every emit mode with every side count, unordered; then one ordered variant (ordered session joins never merge).  Over
# a collapse, whose surviving session holds 2 M values, `running` with 3 or 4 sides and `final` with 4 would expand to
# 10^6 - 10^7 rows; those run on the other builders only.
K16_CASES = [("running", 2, False), ("complete", 3, False)]
K16_CASES += [(e, s, False) for e in ks.sp.EMITS for s in (1, 2, 3, 4) if (e, s, False) not in K16_CASES] + [("final", 2, True)]
K16_HEAVY = {("running", 3), ("running", 4), ("final", 4)}


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_k16_session_builders(ctx, M, builder):
    clock, steps0 = ks.session_builders(M)[builder]
    cases = [c for c in K16_CASES if not (builder.startswith("collapse") and c[:2] in K16_HEAVY)]
    for emit, sides, ordered in _variants(M, cases):
        _k16(ctx, clock, steps0, M, emit, sides, ordered)


# ---------------------------------------------------------------------------
# the same stream through K10, K12 and K16: all three call K10's session walk
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("builder", ks.SESSION_BUILDERS)
def test_cross_kernel_sessions(ctx, M, builder):
    """K12's closed sessions (key, id, open, close, merged ids) and late keys, and K16's meta rows and late keys, equal
    K10's, call by call, up to the first call one of them refuses (K12 may refuse first: only it counts merge
    intervals)."""
    clock, steps0 = ks.session_builders(M)[builder]
    k10, _, fail10 = _k10(ctx, clock, steps0, M, False, 2, ("first", "final"))
    shape = _sessions_of([g[0] for g in k10])
    k12, _ = _k12(ctx, clock, steps0, M, False)
    k16, fail16 = _k16(ctx, clock, steps0, M, "final", 2)
    assert fail16 == fail10 and len(k12) <= len(k10)
    assert [([(r[0], r[1], r[3]) for r in g[0][1]], [r[0] for r in g[0][2]]) for g in k12] == shape[: len(k12)]
    assert _sessions_of([g[0] for g in k16]) == shape


# ---------------------------------------------------------------------------
# engine: run_main(gpu=True) with a key of 64 sessions or windows, at the engine's default per-key limit
# ---------------------------------------------------------------------------


@pytest.fixture
def device_calls(monkeypatch):
    """As tests/test_gpu_keyed_limits.py's fixture, for K12, K14 and K16: small key tables and batches, the per-key
    limit left at its default; records (class, per-key limit, rows) of every device activation."""
    from bytewax_b200 import gpu

    monkeypatch.setenv("BYTEWAX_B200_KEYS", "256")
    monkeypatch.setenv("BYTEWAX_B200_BATCH", "4096")
    monkeypatch.delenv("BYTEWAX_B200_SESSIONS", raising=False)
    calls = []
    for cls in (gpu.SessionCollectWindow, gpu.ProductJoinWindow, gpu.SessionProductJoinWindow):
        orig = cls.apply

        def apply(self, *a, _orig=orig, **k):
            s = self.spec
            calls.append((type(self).__name__, getattr(s, "max_sessions_per_key", None) or s.max_windows_per_key, len(a[0])))
            return _orig(self, *a, **k)

        monkeypatch.setattr(cls, "apply", apply)
    return calls


def test_engine_session_collect_64(device_calls):
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, SessionWindower

    items, n1 = _engine_items(11, False)

    def build():
        clock = EventClock(lambda v: v[0], timedelta(days=1), now_getter=lambda: FROZEN)
        return _engine_flow([[(k, (t, i)) for k, t, i in items]],
                            lambda s: win.collect_window("c", s[0], clock, SessionWindower(timedelta(seconds=1)), ordered=False), n1)

    host, dev = _engine_both(build)
    assert dev == host
    assert _hot(host[2])[0] == 24  # 64 sessions held at once (nothing closes before EOF), 40 bridges each merging two
    assert device_calls and all(c[:2] == ("SessionCollectWindow", 64) for c in device_calls) and device_calls[0][2] == n1


def test_engine_product_join_sliding_64(device_calls):
    """Sliding windows of 64 s every 1 s: the hot key's items all fall in one offset bucket, so each is in 64 windows and
    the key holds 64 until EOF; each light key keeps to its own bucket."""
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, SlidingWindower

    rnd = random.Random(12)
    items = [("hot", ALIGN + timedelta(seconds=100 + rnd.random())) for _ in range(40)]
    items += [(f"k{k}", ALIGN + timedelta(seconds=10 * k + rnd.random())) for k in (rnd.randrange(8) for _ in range(40))]
    rnd.shuffle(items)
    items = [(k, t, i) for i, (k, t) in enumerate(items)]
    sides = [[(k, {"ts": t, "i": i}) for k, t, i in items if i % 2 == s] for s in (0, 1)]

    def build():
        clock = EventClock(lambda v: v["ts"], timedelta(days=1), now_getter=lambda: FROZEN)
        windower = SlidingWindower(timedelta(seconds=64), timedelta(seconds=1), ALIGN)
        return _engine_flow(sides, lambda s: win.join_window("j", clock, windower, *s, insert_mode="product", emit_mode="final",
                                                             ordered=False), 20)

    host, dev = _engine_both(build)
    assert dev == host
    assert _hot(host[2]) == (64, 100)  # windows 37 .. 100
    n0 = sum(k == "hot" for k, _, i in items if i % 2 == 0)
    assert sum(r[0] == "hot" for r in host[0]) == 64 * n0 * (40 - n0)  # each hot window's product of its two sides
    assert device_calls and all(c[:2] == ("ProductJoinWindow", 64) for c in device_calls)


def test_engine_session_product_join_64(device_calls):
    import bytewax_b200.operators.windowing as win
    from bytewax_b200.operators.windowing import EventClock, SessionWindower

    items, n1 = _engine_items(13, False)
    sides = [[(k, {"ts": t, "i": i}) for k, t, i in items if i % 2 == s] for s in (0, 1)]

    def build():
        clock = EventClock(lambda v: v["ts"], timedelta(days=1), now_getter=lambda: FROZEN)
        return _engine_flow(sides, lambda s: win.join_window("j", clock, SessionWindower(timedelta(seconds=1)), *s, insert_mode="product",
                                                             emit_mode="final", ordered=False), n1 // 2)

    host, dev = _engine_both(build)
    assert dev == host
    assert _hot(host[2])[0] == 24
    assert device_calls and all(c[:2] == ("SessionProductJoinWindow", 64) for c in device_calls)
