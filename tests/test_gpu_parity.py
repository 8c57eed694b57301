"""Parity of the CUDA path (through the C ABI) with the oracles.  Needs an H100: -m gpu."""

import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import coracle, pyoracle as po  # noqa: E402  (checker only)

REL_TOL = 1e-6  # north_star: floating folds within 1e-6 relative


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module", params=["stream", "direct"], autouse=True)
def fold_mode(request):
    """Every parity test runs twice: with the streaming path (fused verdict + bucket scatter, shared-memory segment
    fold: the default) and with the direct hash-table kernel alone (BW_STREAM is read when a fold is created)."""
    old = {k: os.environ.get(k) for k in ("BW_STREAM",)}
    os.environ["BW_STREAM"] = "1" if request.param == "stream" else "0"
    yield request.param
    for k, v in old.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _is_float(case):
    return any(isinstance(v, float) for b in case["batches"] for v in b[2])


def _make_fold(ctx, s, is_float, **kw):
    from bytewax_b200 import gpu

    return gpu.WindowFold(
        ctx, s["reduction"], s["length_us"], s["offset_us"], s["align_us"], s["wait_us"],
        val_dtype="f64" if is_float else "i64", ordered=s["ordered"],
        capacity_hint=kw.pop("capacity_hint", 4096), max_batch_rows=kw.pop("max_batch_rows", 1 << 16),
        max_emit_rows=kw.pop("max_emit_rows", 1 << 18), max_late_rows=kw.pop("max_late_rows", 1 << 18), **kw)


def _cmp_vals(red, got, want, is_float, where):
    if red == "mean":
        assert got[1] == want[1], where
        assert got[0] == pytest.approx(want[0], rel=REL_TOL, abs=1e-9), where
    elif is_float and red == "sum":
        assert got == pytest.approx(want, rel=REL_TOL, abs=1e-9), where
    else:
        assert got == want, where


def _check_activation(fold, em, act, spec, is_float, where):
    red = spec["reduction"]
    want_e = [(k, w, p) for k, w, t, p in act if t == "E"]
    want_l = [(k, w, p) for k, w, t, p in act if t == "L"]
    want_m = [(k, w, p) for k, w, t, p in act if t == "M"]
    got_e = em.down(mean=(red == "mean"))
    assert [(k, w) for k, (w, _) in got_e] == [(k, w) for k, w, _ in want_e], where
    for (k, (w, a)), (_, _, p) in zip(got_e, want_e):
        _cmp_vals(red, a, p, is_float, (where, k, w))
    assert [(k, w, v) for k, (w, v) in em.late()] == want_l, where
    # meta stream == window bounds of the closed rows, same order (windowing.py:1087-1093)
    assert [[k, w, list(fold.window_bounds(w))] for k, (w, _) in got_e] == [[k, w, p] for k, w, p in want_m], where


def test_golden_cases_per_activation(ctx, golden_dir):
    with open(os.path.join(golden_dir, "window_fold_cases.json")) as f:
        cases = json.load(f)
    for name, case in cases.items():
        s = case["spec"]
        is_float = _is_float(case)
        fold = _make_fold(ctx, s, is_float)
        for i, (keys, ts, vals) in enumerate(case["batches"]):
            fold.ingest(keys, vals, ts)
            _check_activation(fold, fold.advance(), case["acts"][i], s, is_float, (name, i))
        _check_activation(fold, fold.eof(), case["acts"][-1], s, is_float, (name, "eof"))
        fold.close()


def test_moving_system_clock_per_step(ctx, golden_dir):
    """`bw_fold_set_system_now` + the notify phase of `bw_advance(system_now_us)` against rows the reference's own
    `_WindowLogic` / `_EventClockLogic` produced under a stepping `now_getter` (tests/golden/system_time_cases.json):
    the watermark drifts with the system clock (an item can be late because time passed), idle keys' windows close."""
    with open(os.path.join(golden_dir, "system_time_cases.json")) as f:
        cases = json.load(f)
    woke = 0
    for name, case in cases.items():
        s = case["spec"]
        fold = _make_fold(ctx, s, False)
        for i, step in enumerate(case["steps"]):
            if step[0] == "batch":
                _kind, now, keys, ts, vals = step
                fold.set_system_now(now)
                fold.ingest(keys, vals, ts)
                em = fold.advance()
            else:
                em = fold.advance(system_now_us=step[1])
                woke += len(em.closed_key)
            _check_activation(fold, em, case["acts"][i], s, False, (name, i, step[0]))
        _check_activation(fold, fold.eof(), case["acts"][-1], s, False, (name, "eof"))
        fold.close()
    assert woke > 20


@pytest.mark.parametrize("red,length,offset,wait", [("count", 10, None, 0), ("sum", 10, 5, 2)])
def test_rows_shipped_early_equal_one_sort(ctx, fold_mode, red, length, offset, wait, monkeypatch):
    """Host commits: rows of closed epochs are ordered and copied out on a side stream while later activations run
    (flush_rows); what `bw_advance` hands back must be exactly what ordering everything at the end gives (BW_FLUSH=0).
    Epochs repeat (their rows must not be split across segments) and some rows are late."""
    S = 1_000_000
    A = 1_640_995_200_000_000
    spec = dict(reduction=red, length_us=length * S, offset_us=offset * S if offset else None, align_us=A, wait_us=wait * S, ordered=False)
    batches = _random_batches(77, 14, 20_000, 500, 6 * S, 3 * S, A)
    epochs = [1, 1, 2, 3, 3, 3, 4, 5, 6, 6, 7, 8, 9, 9]
    got = {}
    for flush in ("0", "1"):
        monkeypatch.setenv("BW_FLUSH", flush)
        fold = _make_fold(ctx, spec, False, capacity_hint=2048, max_batch_rows=1 << 15, max_emit_rows=1 << 20, max_late_rows=1 << 20)
        for (keys, ts, vals), ep in zip(batches, epochs):
            fold.ingest(keys, vals, ts, ep)
            fold.sync()  # (the counts of the folded activations reach the host: the next commit ships their rows)
        em, em2 = fold.advance(), fold.eof()
        got[flush] = [np.concatenate([getattr(em, f), getattr(em2, f)]) for f in
                      ("closed_key", "closed_window_id", "closed_acc", "closed_epoch", "late_key", "late_window_id", "late_val", "late_ts_us", "late_epoch")]
        fold.close()
    assert len(got["1"][0]) > 1000 and len(got["1"][4]) > 100
    for a, b in zip(got["0"], got["1"]):
        assert np.array_equal(a, b)


def test_golden_cases_single_advance(ctx, golden_dir):
    """All activations committed back to back, rows collected once: same rows, grouped by epoch."""
    with open(os.path.join(golden_dir, "window_fold_cases.json")) as f:
        cases = json.load(f)
    for name in ("tumbling_count_lates", "sliding_sum_lates", "c1_shape_small", "discard_resets_watermark",
                 "ordered_count_wait", "sliding_count_indivisible_negative"):
        case = cases[name]
        s = case["spec"]
        fold = _make_fold(ctx, s, _is_float(case))
        for keys, ts, vals in case["batches"]:
            fold.ingest(keys, vals, ts)
        em = fold.advance()
        want = [(i + 1, k, w) for i, act in enumerate(case["acts"][:-1]) for k, w, t, _ in act if t == "E"]
        assert list(zip(em.closed_epoch.tolist(), em.closed_key.tolist(), em.closed_window_id.tolist())) == want, name
        _check_activation(fold, fold.eof(), case["acts"][-1], s, _is_float(case), (name, "eof"))
        fold.close()


def _random_batches(seed, nb, n, n_keys, span_us, jitter_us, start):
    rnd = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        base = start + b * span_us + (np.arange(n) * span_us) // n
        ts = base + rnd.integers(-jitter_us, jitter_us + 1, n) if jitter_us else base
        out.append((rnd.integers(0, n_keys, n).astype(np.uint64), ts.astype(np.int64), rnd.integers(-1000, 1000, n)))
    return out


@pytest.mark.parametrize("red,length,offset,wait,jitter,ordered", [
    ("count", 10, None, 0, 0, False),      # in order: fast path only
    ("count", 10, None, 3, 2, False),      # disorder inside the wait: fast path
    ("count", 10, None, 0, 6, False),      # late items: exact path
    ("sum", 10, 5, 1, 4, False),           # sliding + late
    ("max", 7, None, 2, 5, False),
    ("min", 60, 10, 0, 3, False),          # 6 windows per item
    ("count", 10, 3, 2, 2, True),          # ordered, indivisible offset
    ("sum", 10, None, None, 30, False),    # wait forever: everything closes at EOF
])
def test_against_c_oracle_medium(ctx, fold_mode, red, length, offset, wait, jitter, ordered):
    S = 1_000_000
    spec = dict(reduction=red, length_us=length * S, offset_us=offset * S if offset else None,
                align_us=1_640_995_200_000_000, wait_us=None if wait is None else wait * S, ordered=ordered)
    batches = _random_batches(hash((red, length, jitter)) & 0xFFFF, 6, 50_000, 3000, 20 * S, jitter * S, spec["align_us"] - 5 * S)
    orc = coracle.COracle(red, spec["length_us"], spec["offset_us"], spec["align_us"],
                          (1 << 62) if wait is None else wait * S, ordered)
    fold = _make_fold(ctx, spec, False, capacity_hint=8192, max_batch_rows=1 << 16, max_emit_rows=1 << 20, max_late_rows=1 << 21)
    for keys, ts, vals in batches:
        orc.on_batch(keys, ts, vals)
        fold.ingest(keys, vals, ts)
    orc.on_eof()
    em, em_eof = fold.advance(), fold.eof()
    ck, cw, ca, cc, cact = orc.closed()
    lk, lw, lv, lts, lact = orc.late()
    got = np.concatenate
    assert got([em.closed_key, em_eof.closed_key]).tolist() == ck.tolist()
    assert got([em.closed_window_id, em_eof.closed_window_id]).tolist() == cw.tolist()
    assert got([em.closed_acc.astype(np.int64), em_eof.closed_acc.astype(np.int64)]).tolist() == ca.tolist()
    assert em.closed_epoch.tolist() == (cact[: len(em.closed_epoch)] + 1).tolist()
    assert em.late_key.tolist() == lk.tolist() and em.late_window_id.tolist() == lw.tolist()
    assert em.late_val.astype(np.int64).tolist() == lv.tolist() and em.late_ts_us.tolist() == lts.tolist()
    st = fold.stats()
    if jitter > (wait if wait is not None else 10**9):
        assert st.slow_batches + st.split_batches > 0
    if fold_mode == "stream" and wait is not None:  # every clean activation took the streaming path
        assert st.combined_folds == st.fold_launches and st.fold_launches + st.slow_batches == len(batches)
    if fold_mode == "direct":
        assert st.combined_folds == 0
    fold.close()
    orc.close()


@pytest.mark.parametrize("red,length,offset,wait,dtype,shape", [
    ("count", 10, None, 0, "i64", "stragglers"),
    ("sum", 10, None, 2, "i64", "stragglers"),
    ("sum", 10, 5, 1, "i64", "stragglers"),        # sliding: a late row is reported once per window it would have joined
    ("min", 10, None, 2, "i64", "stragglers"),
    ("sum", 10, None, 1, "f64", "stragglers"),
    ("sum", 10, None, 1, "i64", "jump"),           # a row from the future makes the same key's next rows late
    ("count", 10, 5, 1, "i64", "jump"),
    ("max", 10, None, 0, "i64", "first-row"),      # row 0 of every activation is an hour old (base of the relative timestamps)
])
def test_stragglers_without_the_sort(ctx, fold_mode, red, length, offset, wait, dtype, shape):
    """An in-order stream with a few late rows: the streaming path finds them with the suspect table (bw_late.cuh) and
    folds the rest as a clean activation; rows, late rows and their order must be the exact path's (= the oracle's)."""
    S = 1_000_000
    A = 1_640_995_200_000_000
    n, nb, n_keys = 60_000, 6, 4000
    rnd = np.random.default_rng(hash((red, length, shape)) & 0xFFFF)
    is_float = dtype == "f64"
    orc = coracle.COracle(red, length * S, offset * S if offset else None, A, wait * S, False, is_float=is_float)
    fold = _make_fold(ctx, dict(reduction=red, length_us=length * S, offset_us=offset * S if offset else None, align_us=A,
                                wait_us=wait * S, ordered=False), is_float, capacity_hint=8192, max_batch_rows=1 << 16,
                      max_emit_rows=1 << 20, max_late_rows=1 << 20)
    n_dirty = 0
    for b in range(nb):
        keys = rnd.integers(0, n_keys, n).astype(np.uint64)
        ts = (A + b * 8 * S + (np.arange(n) * 8 * S) // n).astype(np.int64)
        if b != 2 and not (shape == "first-row" and b == 0):  # (one activation stays clean; the very first row ever is never late)
            n_dirty += 1
            if shape == "stragglers":
                late = rnd.random(n) < 0.005
                ts[late] -= rnd.integers(3 * S, 40 * S, int(late.sum()))
            elif shape == "jump":
                at = int(rnd.integers(n // 4, n // 2))
                ts[at] += wait * S + S // 2          # the rows of the next half second are behind it by more than `wait`
                keys[at + 1: at + 2000: 7] = keys[at]  # ... and some of them are this key's: late; the others are not
                late = rnd.random(n) < 0.001
                ts[late] -= 20 * S
            else:
                ts[0] -= 3600 * S
                ts[n // 2] -= 3 * S
        vals = rnd.normal(0, 100, n) if is_float else rnd.integers(-1000, 1000, n)
        orc.on_batch(keys, ts, vals)
        fold.ingest(keys, vals, ts)
    orc.on_eof()
    em, em_eof = fold.advance(), fold.eof()
    ck, cw, ca, cc, cact = orc.closed()
    lk, lw, lv, lts, lact = orc.late()
    cat = np.concatenate
    assert len(lk) > 0
    assert cat([em.closed_key, em_eof.closed_key]).tolist() == ck.tolist()
    assert cat([em.closed_window_id, em_eof.closed_window_id]).tolist() == cw.tolist()
    got_acc = cat([em.closed_acc, em_eof.closed_acc])
    if is_float:
        assert np.allclose(got_acc.astype(np.float64), np.asarray(ca, dtype=np.float64), rtol=REL_TOL, atol=1e-9)
    else:
        assert got_acc.astype(np.int64).tolist() == ca.tolist()
    assert em.closed_epoch.tolist() == (cact[: len(em.closed_epoch)] + 1).tolist()
    assert em.late_key.tolist() == lk.tolist() and em.late_window_id.tolist() == lw.tolist()
    assert em.late_ts_us.tolist() == lts.tolist()
    if is_float:
        assert np.array_equal(em.late_val.astype(np.float64), np.asarray(lv, dtype=np.float64))
    else:
        assert em.late_val.astype(np.int64).tolist() == lv.tolist()
    st = fold.stats()
    if fold_mode == "stream":
        assert st.split_batches == n_dirty and st.slow_batches == 0, (st.split_batches, st.slow_batches)
        assert st.combined_folds == nb
    else:
        assert st.slow_batches == n_dirty
    fold.close()
    orc.close()


def test_activation_spanning_several_windows(ctx, fold_mode):
    """In-order activations that each span 3.5 windows: the direct kernel folds them in sub-ranges with a
    close in between (one per pane of event-time span); rows must not change."""
    S = 1_000_000
    A = 1_640_995_200_000_000
    n, nb, n_keys = 1 << 21, 3, 5000
    fold = _make_fold(ctx, dict(reduction="count", length_us=10 * S, offset_us=None, align_us=A, wait_us=2 * S, ordered=False),
                      False, capacity_hint=8192, max_batch_rows=n, max_emit_rows=1 << 20)
    orc = coracle.COracle("count", 10 * S, None, A, 2 * S, False)
    rnd = np.random.default_rng(11)
    for b in range(nb):
        keys = rnd.integers(0, n_keys, n).astype(np.uint64)
        ts = (A + b * 35 * S + (np.arange(n) * 35 * S) // n + rnd.integers(-S, S + 1, n)).astype(np.int64)
        orc.on_batch(keys, ts, np.ones(n, np.int64))
        fold.ingest(keys, None, ts)
    orc.on_eof()
    em, em_eof = fold.advance(), fold.eof()
    ck, cw, ca, _, cact = orc.closed()
    assert np.concatenate([em.closed_key, em_eof.closed_key]).tolist() == ck.tolist()
    assert np.concatenate([em.closed_window_id, em_eof.closed_window_id]).tolist() == cw.tolist()
    assert np.concatenate([em.closed_acc, em_eof.closed_acc]).astype(np.int64).tolist() == ca.tolist()
    assert em.closed_epoch.tolist() == (cact[: len(em.closed_epoch)] + 1).tolist()
    st = fold.stats()
    assert st.slow_batches == 0
    if fold_mode == "direct":
        assert st.fold_launches > nb  # the activations were split
    fold.close()
    orc.close()


def test_float_sum_and_mean_tolerance(ctx):
    S = 1_000_000
    rnd = np.random.default_rng(5)
    for red in ("sum", "mean", "min", "max"):
        for dtype in ("f32", "f64"):
            from bytewax_b200 import gpu

            n = 40_000
            keys = rnd.integers(0, 500, n).astype(np.uint64)
            ts = (1_640_995_200_000_000 + np.arange(n) * 1000).astype(np.int64)
            vals = rnd.random(n).astype(np.float32 if dtype == "f32" else np.float64)
            fold = gpu.WindowFold(ctx, red, 10 * S, None, wait_us=0, val_dtype=dtype, capacity_hint=2048,
                                  max_batch_rows=1 << 16, max_emit_rows=1 << 16)
            orc = coracle.COracle(red, 10 * S, is_float=True)
            for lo in range(0, n, 10_000):
                sl = slice(lo, lo + 10_000)
                fold.ingest(keys[sl], vals[sl], ts[sl])
                orc.on_batch(keys[sl], ts[sl], vals[sl].astype(np.float64))
            orc.on_eof()
            em, em2 = fold.advance(), fold.eof()
            ck, cw, ca, cc, _ = orc.closed()
            gk = np.concatenate([em.closed_key, em2.closed_key])
            ga = np.concatenate([em.closed_acc, em2.closed_acc])
            gc = np.concatenate([em.closed_count, em2.closed_count])
            assert gk.tolist() == ck.tolist()
            if red in ("min", "max"):
                assert ga.tolist() == ca.tolist()  # exact: no rounding in min/max
            else:
                np.testing.assert_allclose(ga, ca, rtol=REL_TOL)
            if red == "mean":
                assert gc.tolist() == cc.tolist()
            fold.close()
            orc.close()


def test_edge_cases(ctx):
    from bytewax_b200 import gpu

    S = 1_000_000
    A = 1_640_995_200_000_000
    fold = gpu.WindowFold(ctx, "count", 10 * S, None, A, 0, capacity_hint=64, max_batch_rows=1024)
    # empty activation
    fold.ingest(np.zeros(0, np.uint64), None, np.zeros(0, np.int64))
    assert fold.advance().closed_key.size == 0
    # key == 2^64-1 (the table's empty sentinel), key 0, 20-digit keys, negative windows
    keys = np.array([2**64 - 1, 0, 2**64 - 1, 10**19, 10**19 + 5, 9, 10, 100, 99], dtype=np.uint64)
    ts = np.array([A - 25 * S] * 9, dtype=np.int64)
    fold.ingest(keys, None, ts)
    em = fold.eof()
    want = sorted(set(keys.tolist()), key=str)
    assert em.closed_key.tolist() == want
    assert em.closed_window_id.tolist() == [-3] * len(want)
    assert dict(zip(em.closed_key.tolist(), em.closed_acc.tolist()))[2**64 - 1] == 2
    fold.close()
    # one key, many windows inside one activation; first-opened order != id order
    fold = gpu.WindowFold(ctx, "count", 10 * S, None, A, 50 * S, capacity_hint=64, max_batch_rows=1024)
    ts = np.array([A + 31 * S, A + 5 * S, A + 12 * S, A + 33 * S, A + 95 * S], dtype=np.int64)
    fold.ingest(np.full(5, 7, np.uint64), None, ts)
    em = fold.advance()
    assert em.closed_window_id.tolist() == [3, 0, 1]  # closed by wm = 45 s, in first-opened order
    assert em.closed_acc.tolist() == [2, 1, 1]
    assert fold.eof().closed_window_id.tolist() == [9]
    fold.close()


def test_errors_are_loud(ctx):
    from bytewax_b200 import _native as N, gpu

    with pytest.raises(N.BwError) as e:
        gpu.WindowFold(ctx, "count", 10, 20)  # offset > length
    assert e.value.status == 4
    fold = gpu.WindowFold(ctx, "count", 10_000_000, capacity_hint=16, max_batch_rows=1 << 16, max_emit_rows=8)
    keys = np.arange(60_000, dtype=np.uint64)
    fold.ingest(keys, None, np.full(60_000, 1_640_995_200_000_000, np.int64))
    with pytest.raises(N.BwError) as e:
        fold.advance()
    assert e.value.status == 3  # table full
    fold.close()


def test_c1_properties_and_sampled_parity(ctx, fold_mode):
    """Config C1 (SURVEY.md 8d) at 2^24 rows x 4 batches: exact multiset vs the C oracle at 2M rows,
    then size-independent checks on the rest (sum of counts == N, per-window totals)."""
    from bytewax_b200 import gpu

    A = 1_640_995_200_000_000
    n_keys, B, nb = 100_000, 1 << 22, 6
    L = 5_000_000  # 5 s windows -> a window closes every ~1.2 batches
    fold = gpu.WindowFold(ctx, "count", L, None, A, 0, val_dtype="u64", ts_from_value=True, capacity_hint=n_keys,
                          max_batch_rows=B, max_emit_rows=1 << 23)
    dk, dv = ctx.dev_alloc(B * 8), ctx.dev_alloc(B * 8)
    orc = coracle.COracle("count", L, align_us=A)
    hk, hv = np.empty(B, np.uint64), np.empty(B, np.uint64)
    rows_got = []
    for b in range(nb):
        fold.gen_c1(dk, dv, b * B, B, n_keys)
        fold.ingest_device(dk, dv, None, B)
        if b < 1:
            fold.sync()
            ctx.d2h(hk, dk)
            ctx.d2h(hv, dv)
            k2, t2, v2 = coracle.gen_c1(b * B, B, n_keys, A)
            assert hk.tolist() == k2.tolist() and hv.tolist() == v2.tolist()
            orc.on_batch(k2, t2)
        em = fold.advance()
        rows_got.append(em)
        if b < 1:
            ck, cw, ca, _, _ = orc.closed()
            assert em.closed_key.tolist() == ck.tolist() and em.closed_window_id.tolist() == cw.tolist()
            assert em.closed_acc.tolist() == ca.tolist()
    rows_got.append(fold.eof())
    total = sum(int(e.closed_acc.sum()) for e in rows_got)
    assert total == nb * B
    wid = np.concatenate([e.closed_window_id for e in rows_got])
    acc = np.concatenate([e.closed_acc for e in rows_got])
    per_window = np.bincount(wid, weights=acc).astype(np.int64)
    nfull = (nb * B) // L
    assert (per_window[:nfull] == L).all() and per_window.sum() == nb * B
    st = fold.stats()
    assert st.slow_batches == 0 and st.fold_launches >= nb
    assert st.combined_folds == (nb if fold_mode == "stream" else 0)
    ctx.dev_free(dk)
    ctx.dev_free(dv)
    fold.close()
    orc.close()


@pytest.mark.parametrize("total_rows", [1 << 20, 10_000_000])
def test_c1_exact_rows_per_activation(ctx, fold_mode, total_rows):
    """Config C1 with its 10^6 distinct keys (SURVEY.md 8d (i)): eight activations, windows scaled so that four close
    before EOF; every activation's rows -- (key, window id, count) AND their order, i.e. the per-key emission
    sequence -- must equal the C oracle's, bit for bit."""
    from bytewax_b200 import gpu

    A = 1_640_995_200_000_000
    n_keys, nb = 1_000_000, 8
    B = total_rows // nb
    L = (total_rows // 4 // 1000) * 1000  # window length in us: the stream spans total_rows us -> ~4 windows
    fold = gpu.WindowFold(ctx, "count", L, None, A, 0, val_dtype="u64", ts_from_value=True, capacity_hint=n_keys,
                          max_batch_rows=B, max_emit_rows=1 << 23)
    dk, dv = ctx.dev_alloc(B * 8), ctx.dev_alloc(B * 8)
    orc = coracle.COracle("count", L, align_us=A)
    got = []
    for b in range(nb):
        fold.gen_c1(dk, dv, b * B, B, n_keys)
        fold.ingest_device(dk, dv, None, B)
        got.append(fold.advance())
        k2, t2, _ = coracle.gen_c1(b * B, B, n_keys, A)
        orc.on_batch(k2, t2)
    got.append(fold.eof())
    orc.on_eof()
    ck, cw, ca, _, cact = orc.closed()
    n_closed_before_eof = 0
    for b in range(nb + 1):
        sel = cact == b
        em = got[b]
        assert np.array_equal(em.closed_key, ck[sel]), (b, len(em.closed_key), int(sel.sum()))
        assert np.array_equal(em.closed_window_id, cw[sel]), b
        assert np.array_equal(em.closed_acc.astype(np.int64), ca[sel]), b
        if b < nb:
            n_closed_before_eof += len(em.closed_key)
    assert n_closed_before_eof > total_rows // 8  # not vacuous: windows closed (per key, by that key's later events) before EOF
    assert sum(int(e.closed_acc.sum()) for e in got) == nb * B
    st = fold.stats()
    assert st.slow_batches == 0
    assert st.combined_folds == (nb if fold_mode == "stream" else 0)
    ctx.dev_free(dk)
    ctx.dev_free(dv)
    fold.close()
    orc.close()


def test_c3_shape_sliding_f32_sum(ctx, fold_mode):
    """Config C3's shape (SURVEY.md 8d): sliding 60 s / 10 s event-time windows, f32 values summed, 10^6 keys, N = 10^6
    rows spread over C3's 1000 s of event time; rows within 1e-6 relative of the oracle (f64 left-to-right sums), and
    the sum over all windows == 6 x the sum of the values (every event lies in six windows)."""
    from bytewax_b200 import gpu

    S = 1_000_000
    A = 1_640_995_200_000_000
    n, n_keys, nb = 1_000_000, 1_000_000, 8
    i = np.arange(n, dtype=np.uint64)

    def sm64(x):  # splitmix64, vectorised (== oracle.pyoracle.splitmix64)
        x = x + np.uint64(0x9E3779B97F4A7C15)
        z = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))

    with np.errstate(over="ignore"):
        keys = sm64(np.uint64(0xC3) ^ i) % np.uint64(n_keys)
        vals = ((sm64(np.uint64(0xF3) ^ i) >> np.uint64(40)).astype(np.float64) / float(1 << 24)).astype(np.float32)
    assert int(keys[5]) == po.splitmix64(0xC3 ^ 5) % n_keys
    ts = (A + np.arange(n, dtype=np.int64) * 1000).astype(np.int64)
    fold = gpu.WindowFold(ctx, "sum", 60 * S, 10 * S, A, 0, val_dtype="f32", capacity_hint=n_keys, max_batch_rows=n // nb,
                          max_emit_rows=1 << 23)
    orc = coracle.COracle("sum", 60 * S, 10 * S, A, 0, False, is_float=True)
    got = []
    for b in range(nb):
        sl = slice(b * (n // nb), (b + 1) * (n // nb))
        fold.ingest(keys[sl], vals[sl], ts[sl])
        orc.on_batch(keys[sl], ts[sl], vals[sl].astype(np.float64))
        got.append(fold.advance())
    got.append(fold.eof())
    orc.on_eof()
    ck, cw, ca, _, cact = orc.closed()
    gk = np.concatenate([e.closed_key for e in got])
    gw = np.concatenate([e.closed_window_id for e in got])
    ga = np.concatenate([e.closed_acc for e in got])
    assert np.array_equal(gk, ck) and np.array_equal(gw, cw)
    np.testing.assert_allclose(ga, ca, rtol=REL_TOL)
    assert abs(float(ga.sum()) - 6.0 * float(vals.astype(np.float64).sum())) <= REL_TOL * 6.0 * float(vals.sum())
    st = fold.stats()
    assert st.slow_batches == 0
    if fold_mode == "stream":
        assert st.combined_folds == nb
    fold.close()
    orc.close()


@pytest.mark.parametrize("red,length,offset,wait", [("count", 10, None, 2), ("sum", 10, 5, 3), ("max", 7, None, 0)])
def test_snapshot_restore_resumes_identically(ctx, red, length, offset, wait):
    """bw_snapshot_take after three activations, bw_snapshot_load into a fresh fold of a different capacity, then the
    same remaining activations through both: identical rows from there on (and equal to the C oracle's), the contract
    of the reference's resume tests (pytests/test_recovery.py, operators/test_stateful.py:151-291) at the fold level."""
    S = 1_000_000
    spec = dict(reduction=red, length_us=length * S, offset_us=offset * S if offset else None,
                align_us=1_640_995_200_000_000, wait_us=wait * S, ordered=False)
    batches = _random_batches(77, 6, 30_000, 2000, 12 * S, min(wait, 2) * S, spec["align_us"] - 3 * S)
    orc = coracle.COracle(red, spec["length_us"], spec["offset_us"], spec["align_us"], wait * S, False)
    a = _make_fold(ctx, spec, False, capacity_hint=8192, max_emit_rows=1 << 20)
    rows_a, rows_b = [], []
    for keys, ts, vals in batches[:3]:
        orc.on_batch(keys, ts, vals)
        a.ingest(keys, vals, ts)
    first = a.advance()
    snap = a.snapshot()
    assert len(snap["key"]) > 0 and snap["batch_no"] == 3
    b = _make_fold(ctx, spec, False, capacity_hint=3000, max_emit_rows=1 << 20)
    b.restore(snap)
    for keys, ts, vals in batches[3:]:
        orc.on_batch(keys, ts, vals)
        a.ingest(keys, vals, ts)
        b.ingest(keys, vals, ts)
    orc.on_eof()
    for f, rows in ((a, rows_a), (b, rows_b)):
        for em in (f.advance(), f.eof()):
            rows.append((em.closed_key.tolist(), em.closed_window_id.tolist(), em.closed_acc.astype(np.int64).tolist(),
                         em.late_key.tolist(), em.late_window_id.tolist()))
    assert rows_a == rows_b
    ck, cw, ca, _, _ = orc.closed()
    got_k = first.closed_key.tolist() + rows_b[0][0] + rows_b[1][0]
    got_w = first.closed_window_id.tolist() + rows_b[0][1] + rows_b[1][1]
    got_a = first.closed_acc.astype(np.int64).tolist() + rows_b[0][2] + rows_b[1][2]
    assert (got_k, got_w, got_a) == (ck.tolist(), cw.tolist(), ca.tolist())
    a.close()
    b.close()
    orc.close()
