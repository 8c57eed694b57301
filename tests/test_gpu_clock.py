"""The window fold's C ABI under a moving system clock, against the oracle.  Needs an H100: -m gpu.

Every stream comes from tests/clock_streams.py, whose shapes tests/test_oracle_clock.py checks on the CPU.  Each runs
three ways -- streaming with the late split (the default), the sort path behind the same scatter (BW_LATE_SPLIT=0) and
the direct kernel (BW_STREAM=0) -- through `bw_fold_set_system_now`, `bw_advance(system_now_us)` and EOF, and per step,
in the device's order, must give the oracle's down rows (key, window, accumulator bits), its late rows (key, window,
value bits, absolute timestamp), and at EOF the keys that survived.  Each activation's path (segment fold, split,
sort) is asserted through `stats()`."""

import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from tests import clock_streams as cs  # noqa: E402

S = cs.S
MODES = ("split", "sort", "direct")


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def default_env(monkeypatch):
    for k in ("BW_STREAM", "BW_LATE_SPLIT", "BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES", "BW_SEG_SHIFT", "BW_FLUSH"):
        monkeypatch.delenv(k, raising=False)


def _set_mode(monkeypatch, mode):
    """Read when a fold is created."""
    monkeypatch.setenv("BW_STREAM", "0" if mode == "direct" else "1")
    monkeypatch.setenv("BW_LATE_SPLIT", "1" if mode == "split" else "0")


# ---------------------------------------------------------------------------- values

F_EDGE = np.array([-0.0, np.inf, -np.inf, 5e-324, 1.5, -2.25, 1.7e308, -1e-300])  # (one zero: DESIGN §10's signed-zero rule)
F32_EDGE = np.array([-0.0, np.inf, -np.inf, 1e-45, 1.5, -2.25, 3.4028235e38, -1e-30], np.float32)
U_EDGE = np.array([0, 1, 2**63 - 1, 2**63, 2**64 - 1, 12345, 2**62, 2**64 - 2], np.uint64)


def values(ids, red, dtype, wrap=False, rough=False):
    """Values for row ids: edge values for min / max / count; for sums, values whose partial sums are exact (so a
    float sum compares bit for bit), values near 2^62 whose i64 sums wrap, or (`rough`) floats of magnitudes 1e-3 ..
    1e3 whose sums round, checked against the binary64 error bound of oracle/exact.py."""
    ids = np.asarray(ids, np.int64)
    h = (ids * 2654435761) % 8
    if red in ("sum", "mean"):
        if rough:
            x = (((ids * 2654435761) % 1000003) / 1000003.0 - 0.5) * 10.0 ** ((ids % 7) - 3)
            return x.astype(np.float32 if dtype == "f32" else np.float64)
        if wrap:
            return (np.int64(2**62) + ids * 977) * np.where(h < 3, -1, 1)
        small = (ids * 7919) % 41 - 20
        return (small * 0.5).astype(np.float32 if dtype == "f32" else np.float64) if dtype in ("f32", "f64") else small
    return {"f64": F_EDGE, "f32": F32_EDGE, "u64": U_EDGE}.get(dtype, U_EDGE.view(np.int64))[h]


def _py(vals, dtype):
    """What the oracle folds: Python ints / floats (f32 widened exactly)."""
    if dtype in ("f32", "f64"):
        return [float(x) for x in np.asarray(vals, np.float64)]
    return [int(x) for x in vals]


def _bits(x, dtype, red):
    if red == "count":
        return int(x)
    if dtype in ("f32", "f64") or red == "mean":
        return int(np.float64(x).view(np.uint64))
    v = int(x) % 2**64  # (i64 sums wrap)
    return v


# ---------------------------------------------------------------------------- the expected rows


_EXPECTED = {}


def expect(case, red, dtype, ordered, wrap=False, rough=False):
    """Per advance (every step but "ingest" / "set_now", then EOF): down rows (key, wid, bits [, count]) and late rows
    (key, wid, value bits, ts); the trace of the run with ids as values tells which row is late.  `rough` sums: the
    down rows carry an exact.FloatSum (exact sum rounded once, sum of magnitudes, count) instead of bits.  (Kept per
    case object: the three modes of a case share it.)"""
    memo = (id(case), red, dtype, ordered, wrap, rough)
    if memo in _EXPECTED:
        return _EXPECTED[memo][1]
    vals = {}
    for st in case.steps:
        if st[0] in ("batch", "ingest"):
            for i, v in zip(st[4].tolist(), values(st[4], red, dtype, wrap, rough)):
                vals[i] = v
    ts_of = {int(i): int(t) for st in case.steps if st[0] in ("batch", "ingest") for i, t in zip(st[4], st[3])}
    if rough:
        from fractions import Fraction

        from oracle import exact

        def frac_of(ids, f=lambda x: x):
            return [Fraction(f(float(v))) for v in np.asarray(values(ids, red, dtype, wrap, rough), np.float64)]

        tr_v = cs.run(case, vals_of=frac_of, red="sum", ordered=ordered)
        tr_a = cs.run(case, vals_of=lambda ids: frac_of(ids, abs), red="sum", ordered=ordered)
        tr_n = cs.run(case, vals_of=lambda ids: [0] * len(ids), red="count", ordered=ordered)
        rows_v = [[(k, w, t, exact.FloatSum(float(p), float(pa), pn) if t == "E" else p)
                   for (k, w, t, p), (_, _, _, pa), (_, _, _, pn) in zip(a, b_, c_)]
                  for a, b_, c_ in zip(tr_v.rows, tr_a.rows, tr_n.rows)]
    else:
        tr_v = cs.run(case, vals_of=lambda ids: _py(values(ids, red, dtype, wrap), dtype), red=red, ordered=ordered)
        rows_v = tr_v.rows
    tr_i = cs.run(case, red="count", ordered=ordered)
    out = []
    for step, rv, ri in zip(case.steps + [("eof",)], rows_v, tr_i.rows):
        if step[0] in ("ingest", "set_now"):
            continue
        down = []
        for k, w, tag, p in rv:
            if tag != "E":
                continue
            if rough:
                down.append((k, w, p))
            else:
                down.append((k, w, _bits(p[0], dtype, red), p[1]) if red == "mean" else (k, w, _bits(p, dtype, red)))
        late = [(k, w, _bits(vals[p], dtype, "x") if dtype in ("f32", "f64") else int(vals[p]) % 2**64, ts_of[p])
                for k, w, tag, p in ri if tag == "L"]
        out.append((down, late))
    _EXPECTED[memo] = (case, (out, tr_v))
    return out, tr_v


def _got(em, red, dtype):
    if red == "mean":
        down = [(int(k), int(w), int(np.float64(a).view(np.uint64)), int(c))
                for k, w, a, c in zip(em.closed_key, em.closed_window_id, em.closed_acc, em.closed_count)]
    else:
        down = [(int(k), int(w), _bits(a, dtype, red)) for k, w, a in zip(em.closed_key, em.closed_window_id, em.closed_acc)]
    if dtype in ("f32", "f64"):
        lv = [int(x) for x in em.late_val.view(np.uint64)]
    else:
        lv = [int(x) % 2**64 for x in em.late_val]
    late = [(int(k), int(w), v, int(t)) for k, w, v, t in zip(em.late_key, em.late_window_id, lv, em.late_ts_us)]
    return down, late


def _expect_path(mode, path):
    """(combined_folds, split_batches, slow_batches) one activation adds (path: clock_streams.activation_paths)."""
    if path == "none":
        return (0, 0, 0)
    if path == "seg":
        return (0, 0, 0) if mode == "direct" else (1, 0, 0)
    if mode == "split" and path == "split":
        return (1, 1, 0)
    return (0, 0, 1)


def run_case(ctx, monkeypatch, mode, case, red=None, dtype="i64", ordered=None, wrap=False, rough=False, check_paths=True,
             capacity_hint=1 << 12, max_emit_rows=1 << 16):
    """The case through one mode; asserts every advance against the oracle.  Returns the stats of the fold."""
    from bytewax_b200 import _native as N
    from bytewax_b200 import gpu

    red = red or case.red
    ordered = case.ordered if ordered is None else ordered
    want, tr = expect(case, red, dtype, ordered, wrap, rough)
    paths = cs.activation_paths(case)
    _set_mode(monkeypatch, mode)
    rows = max([len(s[2]) for s in case.steps if s[0] in ("batch", "ingest")] + [1])
    fold = gpu.WindowFold(ctx, red, case.length, case.offset, case.align, None if case.wait >= cs.FOREVER else case.wait,
                          val_dtype=dtype, ordered=ordered, capacity_hint=capacity_hint, max_batch_rows=rows,
                          max_emit_rows=max_emit_rows, max_late_rows=1 << 16)
    j, prev, pend = 0, (0, 0, 0), (0, 0, 0)
    try:
        for i, st in enumerate(case.steps + [("eof",)]):
            kind = st[0]
            if kind in ("batch", "ingest"):
                fold.set_system_now(st[1])
                fold.ingest(st[2], values(st[4], red, dtype, wrap, rough), st[3])
                pend = tuple(a + b for a, b in zip(pend, _expect_path(mode, paths[i])))
                if kind == "ingest":
                    continue
                em = fold.advance()
            elif kind == "set_now":
                fold.set_system_now(st[1])
                continue
            elif kind == "notify":
                if tr.refuse[i]:
                    with pytest.raises(N.BwError) as e:
                        fold.advance(system_now_us=st[1])
                    assert e.value.status == N.BW_ERR_STATE and "ahead of the system clock" in str(e.value)
                    assert ordered != case.ordered or i == case.refuse_at
                    return None
                em = fold.advance(system_now_us=st[1])
            else:
                em = fold.eof()
            got = _got(em, red, dtype)
            if rough:  # (the order of the device's additions is its own: within the bound of any order)
                assert [(k, w) for k, w, _a in got[0]] == [(k, w) for k, w, _x in want[j][0]], (case.name, mode, i, kind)
                for a, x in zip(em.closed_acc.tolist(), [x for _k, _w, x in want[j][0]]):
                    assert abs(a - x.fsum) <= x.bound(), (case.name, mode, i, kind, a, x)
            else:
                assert got[0] == want[j][0], (case.name, mode, i, kind, "down")
            assert got[1] == want[j][1], (case.name, mode, i, kind, "late")
            st_ = fold.stats()
            cur = (st_.combined_folds, st_.split_batches, st_.slow_batches)
            d = tuple(c - p for c, p in zip(cur, prev))
            if check_paths and kind != "eof":
                assert d == pend, (case.name, mode, i, d, pend)
            prev, pend, j = cur, (0, 0, 0), j + 1
        assert case.refuse_at is None or not ordered
        assert set(int(k) for k in em.closed_key) == tr.live_after[-1]  # the keys that survived to EOF
        return fold.stats()
    finally:
        fold.close()


# ---------------------------------------------------------------------------- every builder, three ways


@pytest.mark.parametrize("case,mode", [pytest.param(c, m, id=f"{c.name}-{m}") for c in cs.all_cases() for m in MODES])
def test_builder_three_ways(ctx, monkeypatch, case, mode):
    """(wall_clock_2026_ordered on the split: a key woken by its late rows whose pane K4 moved into pane 1 lost it --
    a fold that orders by window id keeps no arrival sequence, and pane 1 is present iff its sequence is not ~0.)"""
    run_case(ctx, monkeypatch, mode, case)


@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("name", ["key_states", "wall_clock_2026"])
def test_float_sums_within_the_bound(ctx, monkeypatch, name, ordered, dtype):
    """f32 / f64 sums that round, three ways: every window's sum within the binary64 error bound of any summation
    order around the exact sum (oracle/exact.py); late rows keep their value bits."""
    case = {"key_states": cs.key_states, "wall_clock_2026": lambda: cs.wall_clock_2026(False)}[name]()
    for mode in MODES:
        run_case(ctx, monkeypatch, mode, case, red="sum", dtype=dtype, ordered=ordered, rough=True)


# ---------------------------------------------------------------------------- reductions and value types

REDS = ([("count", d, False) for d in ("i64", "u64", "f32", "f64")]
        + [(r, d, False) for r in ("min", "max") for d in ("i64", "u64", "f32", "f64")]
        + [("sum", "i64", True), ("sum", "f64", False), ("sum", "f32", False), ("mean", "f64", False)])


@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("red,dtype,wrap", REDS)
@pytest.mark.parametrize("name", ["key_states", "drift", "sliding_partial_10_4"])
def test_reductions_under_a_moving_clock(ctx, monkeypatch, name, red, dtype, wrap, ordered):
    """count, min and max over every value type bit for bit (infinities, denormals, -0.0, u64 above 2^63), i64 sums
    that wrap, f32 / f64 sums and means whose partial sums are exact; unordered and ordered; three ways."""
    case = {"key_states": cs.key_states, "drift": cs.drift, "sliding_partial_10_4": lambda: cs.sliding_partial(10 * S, 4 * S)}[name]()
    for mode in MODES:
        run_case(ctx, monkeypatch, mode, case, red=red, dtype=dtype, ordered=ordered, wrap=wrap)


# ---------------------------------------------------------------------------- many keys, many segments


def _sm_count():
    import ctypes as C

    cu = C.CDLL("libcuda.so.1")
    dev, n = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0
    return n.value


@pytest.mark.parametrize("n_keys,frac", [(100_000, 0.01), (100_000, 0.5), (100_000, 1.0), (1_000_000, 0.5)])
def test_many_keys_many_passes(ctx, monkeypatch, n_keys, frac):
    """10^5 and 10^6 random u64 keys over a table of 2^19+ slots in many segments -- more than k_close_wake's grid
    (8 blocks of 256 per SM), so its grid-stride loop runs more than one pass -- with 1 %, 50 % or all of them due."""
    case = cs.many_keys(n_keys, frac, seed=int(frac * 100))
    cap = 1 << 19 if n_keys <= 100_000 else 1 << 21
    if n_keys > 100_000:  # (the vectorised reference, checked against the oracle at 2 x 10^4 keys)
        want = cs.many_keys_reference(case)
        tr = cs.Trace(refuse=[False, False], live_after=[set(), {k for k, _w, _c in want[-1][0]}])
        _EXPECTED[(id(case), "count", "i64", False, False, False)] = (case, (want, tr))
    for mode in MODES:
        st = run_case(ctx, monkeypatch, mode, case, capacity_hint=cap, max_emit_rows=2 * n_keys)
        assert st.table_capacity + 1 > 8 * 256 * _sm_count()


# ---------------------------------------------------------------------------- C1 size, a notify phase between activations


@functools.lru_cache(maxsize=1)
def _c1_case():
    case = cs.c1_stepping(1 << 22, 1_000_000, 4, seed=7)
    return case, cs.c1_reference(case)


@pytest.mark.parametrize("mode", MODES)
def test_c1_size_stepping_clock(ctx, monkeypatch, mode):
    """2^22 rows per activation over 10^6 keys, the clock stepping 0.7 s per activation (rows at their arrival time, 1 %
    straggling 0.5 .. 2 s back) and a notify phase between every two activations: every step's down and late rows
    against the reference (clock_streams.c1_reference, itself checked against the oracle), and every activation's
    path: the split (the sort path with the split off, or behind the direct kernel)."""
    from bytewax_b200 import gpu

    n = 1 << 22
    case, want = _c1_case()
    _set_mode(monkeypatch, mode)
    fold = gpu.WindowFold(ctx, "count", S, None, cs.A, 0, val_dtype="i64", capacity_hint=1 << 20, max_batch_rows=n,
                          max_emit_rows=1 << 21, max_late_rows=1 << 17)
    prev, g, n_late = (0, 0, 0), -(2**63), 0
    try:
        for i, st in enumerate(case.steps + [("eof",)]):
            if st[0] == "batch":
                fold.set_system_now(st[1])
                fold.ingest(st[2], st[4], st[3])
                em = fold.advance()
                rel = st[3] - st[1]
                runmax = np.maximum.accumulate(np.concatenate([[g], rel[:-1]]))
                n_sus = int((rel < runmax).sum())
                g = max(g, int(rel.max()))
                path = "seg" if n_sus == 0 else ("split" if n_sus <= n // 16 else "sort")
                s_ = fold.stats()
                cur = (s_.combined_folds, s_.split_batches, s_.slow_batches)
                assert tuple(c - p for c, p in zip(cur, prev)) == _expect_path(mode, path), (mode, i, path)
                prev = cur
            elif st[0] == "notify":
                em = fold.advance(system_now_us=st[1])
            else:
                em = fold.eof()
            down, late = want[i]
            got = list(zip(em.closed_key.tolist(), em.closed_window_id.tolist(), em.closed_acc.tolist()))
            assert got == down, (mode, i, len(got), len(down))
            gl = list(zip(em.late_key.tolist(), em.late_window_id.tolist(), em.late_val.tolist(), em.late_ts_us.tolist()))
            assert gl == late, (mode, i, len(gl), len(late))
            n_late += len(late)
    finally:
        fold.close()
    assert n_late > 100_000 and sum(len(d) for d, _ in want) > 2_500_000


# ---------------------------------------------------------------------------- the emit buffer, and EOF


@pytest.mark.parametrize("mode", MODES)
def test_notify_fills_the_emit_buffer(ctx, monkeypatch, mode):
    """max_emit_rows equal to what one notify phase closes passes; one row less is BW_ERR_CAPACITY."""
    from bytewax_b200 import _native as N

    case = cs.emit_capacity()
    run_case(ctx, monkeypatch, mode, case, max_emit_rows=128)
    with pytest.raises(N.BwError) as e:
        run_case(ctx, monkeypatch, mode, case, max_emit_rows=127)
    assert e.value.status == 3


def test_notify_after_eof_is_empty(ctx):
    from bytewax_b200 import gpu

    fold = gpu.WindowFold(ctx, "count", 10 * S, None, cs.A, 0, val_dtype="i64", capacity_hint=1024, max_batch_rows=16)
    try:
        fold.set_system_now(cs.A + 100 * S)
        fold.ingest(np.array([1, 2], np.uint64), np.array([0, 0]), np.array([cs.A + 95 * S, cs.A + 99 * S]))
        assert len(fold.advance().closed_key) == 0
        assert len(fold.eof().closed_key) == 2
        em = fold.advance(system_now_us=cs.A + 1000 * S)
        assert len(em.closed_key) == 0 and len(em.late_key) == 0
    finally:
        fold.close()
