"""Snapshot and restore of the window fold (`bw_snapshot_take` / `bw_snapshot_load`, bw_snapshot.cuh) at every cut, on
every table structure, value type, clock, path and world size.  Needs an H100: -m gpu.

Every resume case runs the stream three ways and compares them per activation:
- uninterrupted: fold A runs the whole stream;
- resumed: fold B restores A's snapshot at the cut and runs the rest; its rows after the cut must be A's;
- oracle: both must match an independent oracle -- the reference's own rows (the golden `acts`), the C oracle for large
  and random streams, oracle/exact.py for float sums and means, u64 and wrapping i64.
Integers, counts and min / max must match bit for bit; float sums and means stay within the error bound of binary64
summation in any order (`exact.FloatSum.bound`).  The last test converts real device snapshots into the reference's
`_WindowSnapshot` (bytewax_b200/snapshot_rows.py) and compares them with what the reference's own `_WindowLogic.snapshot()`
held at the same cut (tests/golden/snapshot_cases.json)."""

import json
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import coracle, exact, pyoracle as po, streams  # noqa: E402  (checker only)

S = 1_000_000
A = 1_640_995_200_000_000
I64_MIN = -(2**63)
KEY_MAX = 2**64 - 1   # the table's empty sentinel: such a key lives in the alias slot `cap`
SEG = 4096            # slots per table segment (BW_SEG_SHIFT_DEFAULT); probe chains wrap inside one
MAX_PANES = 64        # BW_MAX_PANES: live panes per key that the close pass can re-rank
FLOAT = ("f32", "f64")
SNAP_COLS = ("key", "pane_id", "acc", "count", "open_seq", "max_ts_us", "closed_upto")
REL_TOL = 1e-6        # golden float rows: the reference's left-to-right sums, as in test_gpu_parity.py


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module", params=["stream", "direct"], autouse=True)
def fold_mode(request):
    """Every test runs with the streaming path (BW_STREAM=1, the default) and with the direct kernel alone (BW_STREAM=0);
    the variable is read when a fold is created."""
    old = os.environ.get("BW_STREAM")
    os.environ["BW_STREAM"] = "1" if request.param == "stream" else "0"
    yield request.param
    if old is None:
        os.environ.pop("BW_STREAM", None)
    else:
        os.environ["BW_STREAM"] = old


@pytest.fixture(autouse=True)
def default_env(monkeypatch):
    for k in ("BW_LATE_SPLIT", "BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES", "BW_SEG_SHIFT", "BW_FLUSH"):
        monkeypatch.delenv(k, raising=False)


# ---------------------------------------------------------------------------- folds, streams, rows, snapshots


def _spec(red, length, offset=None, wait=0, ordered=False):
    return dict(reduction=red, length_us=length, offset_us=offset, align_us=A, wait_us=wait, ordered=ordered)


def _make(ctx, spec, dtype="i64", cap=4096, rows=1 << 12, emit=1 << 14, late=1 << 14, **kw):
    from bytewax_b200 import gpu

    return gpu.WindowFold(ctx, spec["reduction"], spec["length_us"], spec["offset_us"], spec["align_us"], spec["wait_us"],
                          val_dtype=dtype, ordered=spec["ordered"], capacity_hint=cap, max_batch_rows=rows,
                          max_emit_rows=emit, max_late_rows=late, **kw)


def _batches(batches, now=None):
    """Steps of a frozen-clock stream."""
    return [("batch", now, k, t, v) for k, t, v in batches]


def _play(fold, steps):
    """One step: ("batch", system now or None, keys, ts, vals) ingests and advances; ("notify", now) advances at `now`."""
    out = []
    for st in steps:
        if st[0] == "batch":
            _, now, keys, ts, vals = st
            if now is not None:
                fold.set_system_now(now)
            fold.ingest(keys, vals, ts)
            out.append(fold.advance())
        else:
            out.append(fold.advance(system_now_us=st[1]))
    return out


def _uninterrupted(ctx, spec, steps, dtype="i64", **kw):
    """Fold A over the whole stream: the rows of every step and EOF, and its snapshot before the first step and after
    every step (snapshots[c] is the state at cut c)."""
    a = _make(ctx, spec, dtype, **kw)
    try:
        snaps, ems = [a.snapshot()], []
        for st in steps:
            ems += _play(a, [st])
            snaps.append(a.snapshot())
        ems.append(a.eof())
    finally:
        a.close()
    return ems, snaps


def _n_rows(em):
    return len(em.closed_key) + len(em.late_key)


def _resumed(ctx, spec, steps, snap, cut, dtype="i64", **kw):
    """Fold B: a fresh fold restores `snap` and runs steps[cut:] and EOF.  Restoring emits nothing: the close pass that
    re-ranks the restored keys runs at load, and an advance right after it has no row."""
    b = _make(ctx, spec, dtype, **kw)
    try:
        b.restore(snap)
        assert _n_rows(b.advance()) == 0, cut
        ems = _play(b, steps[cut:])
        ems.append(b.eof())
    finally:
        b.close()
    return ems


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64).tolist() if a.dtype.itemsize == 8 else a.tolist()


def _row_cols(em, fuzzy=False):
    """Every column of an emission; `fuzzy` leaves out the accumulator (float sums and means are checked against their
    error bound instead: atomic float adds may associate differently in A and in B)."""
    cols = [em.closed_key.tolist(), em.closed_window_id.tolist(), em.closed_count.tolist(), em.closed_epoch.tolist(),
            em.late_key.tolist(), em.late_window_id.tolist(), _bits(em.late_val), em.late_ts_us.tolist(), em.late_epoch.tolist()]
    if not fuzzy:
        cols.append(_bits(em.closed_acc))
    return cols


def _same_rows(ems_a, ems_b, fuzzy, where):
    assert len(ems_a) == len(ems_b), where
    for j, (ea, eb) in enumerate(zip(ems_a, ems_b)):
        assert _row_cols(ea, fuzzy) == _row_cols(eb, fuzzy), (where, j)


def _canon(snap):
    order = np.lexsort((snap["pane_id"], snap["key"]))
    return {n: snap[n][order].tolist() for n in SNAP_COLS}, (snap["batch_no"], snap["gmax_ts_us"], snap["last_epoch"])


def _same_snapshot(a, b, where):
    """Equal as a multiset of rows (sorted by key, pane): every column exact, and the three scalars."""
    ca, sa = _canon(a)
    cb, sb = _canon(b)
    assert sa == sb, (where, sa, sb)
    for n in SNAP_COLS:
        assert ca[n] == cb[n], (where, n)


def _panes_by_key(snap):
    """{key: [pane ids in the order the snapshot lists them]}: one thread writes a key's rows together, hot pane first,
    then pane 1, then the overflow list."""
    out = {}
    for k, q in zip(snap["key"].tolist(), snap["pane_id"].tolist()):
        out.setdefault(k, []).append(q)
    return out


# ---------------------------------------------------------------------------- oracles


def _check_golden(em, act, spec, is_float, where):
    """One emission against the reference's rows of that activation: (key, window, acc), late (key, window, value) and
    the meta rows' window bounds, in order."""
    red = spec["reduction"]
    want_e = [(k, w, p) for k, w, t, p in act if t == "E"]
    got_e = em.down(mean=(red == "mean"))
    assert [(k, w) for k, (w, _) in got_e] == [(k, w) for k, w, _ in want_e], where
    for (k, (w, a)), (_, _, p) in zip(got_e, want_e):
        if red == "mean":
            assert a[1] == p[1] and a[0] == pytest.approx(p[0], rel=REL_TOL, abs=1e-9), (where, k, w)
        elif is_float and red == "sum":
            assert a == pytest.approx(p, rel=REL_TOL, abs=1e-9), (where, k, w)
        else:
            assert a == p, (where, k, w)
    assert [(k, w, v) for k, (w, v) in em.late()] == [(k, w, p) for k, w, t, p in act if t == "L"], where
    off = spec["offset_us"] or spec["length_us"]
    want_m = [[k, w, p] for k, w, t, p in act if t == "M"]
    assert [[k, w, [A + w * off, A + w * off + spec["length_us"]]] for k, (w, _) in got_e] == want_m, where


def _check_coracle(ems, want, where, acc=True):
    """Emissions against the C oracle's rows, per activation (`want`: its closed() and late() columns)."""
    ck, cw, ca, cc, cact = want["closed"]
    lk, lw, lv, lts, lact = want["late"]
    for b, e in enumerate(ems):
        sel = cact == b
        assert e.closed_key.tolist() == ck[sel].tolist() and e.closed_window_id.tolist() == cw[sel].tolist(), (where, b)
        if acc:
            assert e.closed_acc.astype(np.int64).tolist() == ca[sel].astype(np.int64).tolist(), (where, b)
        sel = lact == b
        assert e.late_key.tolist() == lk[sel].tolist() and e.late_window_id.tolist() == lw[sel].tolist(), (where, b)
        assert e.late_ts_us.tolist() == lts[sel].tolist(), (where, b)
        if acc:
            assert e.late_val.astype(np.int64).tolist() == lv[sel].astype(np.int64).tolist(), (where, b)


def _coracle(spec, batches, is_float=False):
    orc = coracle.COracle(spec["reduction"], spec["length_us"], spec["offset_us"], A, spec["wait_us"], spec["ordered"],
                          is_float=is_float)
    try:
        for keys, ts, vals in batches:
            orc.on_batch(keys, ts, vals)
        orc.on_eof()
        return dict(closed=orc.closed(), late=orc.late())
    finally:
        orc.close()


def _after(want, cut):
    """The oracle's rows of activations `cut` onwards, numbered from 0."""
    ck, cw, ca, cc, cact = want["closed"]
    lk, lw, lv, lts, lact = want["late"]
    c, l = cact >= cut, lact >= cut
    return dict(closed=(ck[c], cw[c], ca[c], cc[c], cact[c] - cut), late=(lk[l], lw[l], lv[l], lts[l], lact[l] - cut))


def _inorder(rnd, n, n_keys, t0, span=8 * S):
    keys = rnd.integers(0, n_keys, n).astype(np.uint64)
    ts = (t0 + (np.arange(n) * span) // n).astype(np.int64)
    return keys, ts


def _straggle(keys, ts, at, back=40 * S):
    at = np.asarray(at)
    keys[at] = keys[at - 1]
    ts[at] = ts[at - 1] - back


def _apart(rnd, n, k):
    return np.sort(rnd.choice(np.arange(2, n, 2), k, replace=False))


# ---------------------------------------------------------------------------- 1. every cut of every golden case


def _golden_steps(case):
    if "steps" in case:
        return [tuple(s) for s in case["steps"]]
    return _batches(case["batches"])


@pytest.mark.parametrize("file", ["window_fold_cases.json", "system_time_cases.json"])
def test_every_cut_of_every_golden_case(ctx, golden_dir, file):
    """Cut after every activation (0 .. n) of every golden case; even cuts restore into a table of one segment (smaller
    than A's two), odd cuts into one of four (larger), so every case restores into both sizes.  Under the moving clock B gets the same set-now and notify steps after the cut.  A
    stream of hundreds of one-row activations is followed for 2 steps past each cut, and then B's state must equal A's."""
    with open(os.path.join(golden_dir, file)) as f:
        cases = json.load(f)
    n_cuts = 0
    for name, case in cases.items():
        spec = case["spec"]
        is_float = any(isinstance(v, float) for s in _golden_steps(case) if s[0] == "batch" for v in s[4])
        dtype = "f64" if is_float else "i64"
        fuzzy = is_float and spec["reduction"] in ("sum", "mean")
        steps = _golden_steps(case)
        ems_a, snaps = _uninterrupted(ctx, spec, steps, dtype)
        for i, em in enumerate(ems_a):
            _check_golden(em, case["acts"][i], spec, is_float, (name, "A", i))
        horizon = len(steps) if len(steps) <= 40 else 2
        for cut in range(len(steps) + 1):
            end = min(len(steps), cut + horizon)
            for cap in ((16, 6000)[cut % 2],):
                if end < len(steps):
                    b = _make(ctx, spec, dtype, cap=cap)
                    try:
                        b.restore(snaps[cut])
                        assert _n_rows(b.advance()) == 0
                        got = _play(b, steps[cut:end])
                        _same_snapshot(b.snapshot(), snaps[end], (name, cut, cap))
                    finally:
                        b.close()
                else:
                    got = _resumed(ctx, spec, steps, snaps[cut], cut, dtype, cap=cap)
                _same_rows(ems_a[cut:cut + len(got)], got, fuzzy, (name, cut, cap))
                for j, em in enumerate(got):
                    _check_golden(em, case["acts"][cut + j], spec, is_float, (name, cut, cap, j))
                n_cuts += 1
    assert n_cuts > 60


# ---------------------------------------------------------------------------- 2. chained restores


@pytest.mark.parametrize("name", ["random", "random_clock_sum_1"])
def test_chained_restores(ctx, golden_dir, name):
    """After every activation the state moves into a fresh fold (alternating table sizes), which runs the next
    activation: the rows must equal the uninterrupted run's.  At every link take(restore(take(A))) == take(A)."""
    if name == "random":
        spec = _spec("sum", 10 * S, 5 * S, 2 * S)
        rnd = np.random.default_rng(21)
        batches = []
        for b in range(10):
            keys, ts = _inorder(rnd, 8000, 700, A + b * 6 * S, 6 * S)
            ts = ts + rnd.integers(-3 * S, 3 * S, len(ts))
            batches.append((keys, ts, rnd.integers(-1000, 1000, len(ts))))
        steps = _batches(batches)
        want = _coracle(spec, batches)
        assert len(want["late"][0]) > 50
    else:
        with open(os.path.join(golden_dir, "system_time_cases.json")) as f:
            case = json.load(f)[name]
        spec, steps = case["spec"], _golden_steps(case)
    ems_a, _ = _uninterrupted(ctx, spec, steps, rows=1 << 13)
    fold = _make(ctx, spec, rows=1 << 13)
    got = []
    try:
        for i, st in enumerate(steps):
            got += _play(fold, [st])
            snap = fold.snapshot()
            nxt = _make(ctx, spec, cap=[64, 3000][i % 2], rows=1 << 13)
            fold.close()
            fold = nxt
            fold.restore(snap)
            _same_snapshot(fold.snapshot(), snap, (name, i))
        got.append(fold.eof())
    finally:
        fold.close()
    _same_rows(ems_a, got, False, name)
    if name == "random":
        _check_coracle(got, want, name)
    else:
        for i, em in enumerate(got):
            _check_golden(em, case["acts"][i], spec, False, (name, i))


# ---------------------------------------------------------------------------- 3. table structures at the cut


def _resume_every_cut(ctx, spec, batches, dtype="i64", want=None, fuzzy=False, **kw):
    """A over `batches`, B from every cut; A == oracle and B == A after the cut.  Returns A's snapshots."""
    steps = _batches(batches)
    ems_a, snaps = _uninterrupted(ctx, spec, steps, dtype, **kw)
    if want is not None:
        _check_coracle(ems_a, want, "A", acc=not fuzzy)
    for cut in range(1, len(steps) + 1):
        got = _resumed(ctx, spec, steps, snaps[cut], cut, dtype, **kw)
        _same_rows(ems_a[cut:], got, fuzzy, cut)
    return snaps


@pytest.mark.parametrize("k4_panes", [MAX_PANES - 1, MAX_PANES])
def test_pane_structures_at_the_cut(ctx, k4_panes):
    """Keys holding, at the cut: two adjacent panes in the direct slots, three and more live panes (overflow nodes),
    BW_MAX_PANES - 1 and exactly BW_MAX_PANES live panes on one key (resumed through EOF, whose close pass gathers them
    all), and keys 0 and 2^64-1 (the alias slot) with several panes.  Pane 1 is always the pane BEFORE pane 0 at a cut
    (`p1_prev`), whichever arrived first: the close pass, which runs on every key an activation creates a pane for and on
    every restored key, puts the newest pane in the hot slot; the "pane 1 = pane 0 + 1" form only lives inside an
    activation.  A row that brings a key with BW_MAX_PANES live panes a 65th one stops the fold with BW_ERR_CAPACITY
    (DESIGN.md section 10): loudly, never a silent drop."""
    spec = _spec("sum", S, None, 100 * S)   # 1 s tumbling windows, 100 s wait: nothing closes for a while
    t0 = A + 1000 * S
    keys, ts = [], []

    def add(k, secs):
        keys.extend([k] * len(secs))
        ts.extend(t0 + int(x * S) for x in secs)

    add(1, [0.1, 1.2])             # pane 0 then the next one
    add(2, [1.3, 0.4])             # a newer pane first, then the one before it
    add(3, [0.5, 1.5, 2.5, 3.5])   # overflow list
    add(4, [i + 0.25 for i in range(k4_panes)])  # up to exactly BW_MAX_PANES live panes
    add(0, [0.6, 1.6, 2.6])
    add(KEY_MAX, [0.7, 2.7, 1.7, 5.7])
    rnd = np.random.default_rng(3)
    b0 = (np.array(keys, np.uint64), np.array(ts, np.int64), rnd.integers(-50, 50, len(keys)))
    b1 = (np.array([1, 2, 3, 4, 0, KEY_MAX, 5], np.uint64), np.array([t0 + 70 * S] * 3 + [t0 + 10 * S + S // 2] + [t0 + 70 * S] * 3, np.int64),
          rnd.integers(-50, 50, 7))  # (key 4 stays at BW_MAX_PANES)
    # (key 4 gets no row after b1: its panes stay live to EOF, whose close pass gathers all of them)
    b2 = (np.array([1, 2, 3, 0, KEY_MAX], np.uint64), np.full(5, t0 + 500 * S, np.int64), rnd.integers(-50, 50, 5))
    batches = [b0, b1, b2]
    snaps = _resume_every_cut(ctx, spec, batches, want=_coracle(spec, batches))
    p0 = (t0 - A) // S
    panes = _panes_by_key(snaps[1])
    # the close pass leaves the newest pane in the hot slot and the one before it in pane 1, whichever arrived first
    assert panes[1] == [p0 + 1, p0] and panes[2] == [p0 + 1, p0]
    assert sorted(panes[3]) == [p0 + i for i in range(4)]
    assert sorted(panes[4]) == [p0 + i for i in range(k4_panes)]
    assert sorted(panes[0]) == [p0, p0 + 1, p0 + 2] and sorted(panes[KEY_MAX]) == [p0, p0 + 1, p0 + 2, p0 + 5]
    panes = _panes_by_key(snaps[2])
    assert len(panes[4]) == k4_panes and sorted(panes[3]) == [p0 + i for i in range(4)] + [p0 + 70]
    assert len(_panes_by_key(snaps[3])[4]) == k4_panes and len(_panes_by_key(snaps[3])[3]) == 1
    if k4_panes == MAX_PANES:
        # a row for a 65th pane: the close pass of that activation gathers 65 panes and stops the fold loudly
        from bytewax_b200 import _native as N

        b = _make(ctx, spec)
        try:
            b.restore(snaps[1])
            with pytest.raises(N.BwError) as e:
                b.ingest(np.array([4], np.uint64), np.array([1]), np.array([t0 + 80 * S], np.int64))
                b.advance()
            assert e.value.status == 3
        finally:
            b.close()


def test_sliding_overflow_panes(ctx):
    """Sliding 60 s / 10 s windows (6 panes per window) with a 30 s wait and disorder inside it: most keys hold 3+ live
    panes at every cut, in overflow nodes."""
    spec = _spec("count", 60 * S, 10 * S, 30 * S)
    rnd = np.random.default_rng(4)
    batches = []
    for b in range(6):
        keys, ts = _inorder(rnd, 20_000, 500, A + b * 25 * S, 25 * S)
        batches.append((keys, ts + rnd.integers(-20 * S, 20 * S, len(ts)), None))
    snaps = _resume_every_cut(ctx, spec, batches, want=_coracle(spec, [(k, t, np.zeros(len(k), np.int64)) for k, t, _ in batches]),
                              rows=20_000)
    for c in range(1, 6):
        counts = np.bincount(np.unique(snaps[c]["key"], return_inverse=True)[1])
        assert (counts >= 3).mean() > 0.5, c


def test_discarded_key_and_empty_snapshot(ctx, golden_dir):
    """A key whose windows all closed is discarded (its watermark with it): it is not in the snapshot, and after a
    restore its older rows are not late.  A snapshot of a table with no key (n = 0) still carries batch_no, gmax and the
    last epoch."""
    with open(os.path.join(golden_dir, "system_time_cases.json")) as f:
        case = json.load(f)["idle_key_closes_on_notify"]
    steps = _golden_steps(case)
    ems, snaps = _uninterrupted(ctx, case["spec"], steps)
    seen = set(int(k) for k in steps[0][2])
    assert seen and seen - set(snaps[-1]["key"].tolist()) == seen  # every key gone by the last notify
    last = snaps[-1]
    assert len(last["key"]) == 0 and last["batch_no"] == 1 and last["gmax_ts_us"] > I64_MIN and last["last_epoch"] == 1
    b = _make(ctx, case["spec"])
    try:
        b.restore(last)
        _same_snapshot(b.snapshot(), last, "empty")
        # the discarded keys come back with rows far behind their old maximum: not late
        k = np.array(sorted(seen), np.uint64)
        b.ingest(k, np.ones(len(k), np.int64), np.full(len(k), min(steps[0][3]) - 60 * S, np.int64))
        em = b.advance()
        assert len(em.late_key) == 0
        em = b.eof()
        assert sorted(em.closed_key.tolist()) == sorted(seen) and len(em.late_key) == 0
    finally:
        b.close()


# ---------------------------------------------------------------------------- 4. value types


def _exact_resume(ctx, red, dtype, vals_fn, length=10 * S, offset=None, wait=3 * S, cuts=(2, 4), seed=0, n=20_000, nb=6):
    """An in-order stream (nothing late, so oracle/exact.py applies) cut at `cuts`: A and every B against the C
    oracle's rows (keys, windows, order, epochs) and oracle/exact.py's accumulators."""
    rnd = np.random.default_rng(seed)
    spec = _spec(red, length, offset, wait)
    batches = []
    for b in range(nb):
        keys, ts = _inorder(rnd, n, 300, A + b * 8 * S)
        batches.append((keys, ts, vals_fn(rnd, n)))
    want = _coracle(_spec("count", length, offset, wait), [(k, t, None) for k, t, _ in batches])
    ex = exact.fold(red, length, offset, A, wait, batches, dtype)
    fuzzy = red == "mean" or (red == "sum" and dtype in FLOAT)
    steps = _batches(batches)
    ems_a, snaps = _uninterrupted(ctx, spec, steps, dtype, rows=n, emit=1 << 16)

    def check(ems, first, where):
        _check_coracle(ems, _after(want, first), where, acc=False)
        k = np.concatenate([e.closed_key for e in ems]).tolist()
        w = np.concatenate([e.closed_window_id for e in ems]).tolist()
        acc = np.concatenate([e.closed_acc for e in ems])
        exp = [ex[kw] for kw in zip(k, w)]
        if fuzzy:
            fs = np.array([x.fsum for x in exp])
            assert (np.abs(acc - fs) <= np.array([x.bound() for x in exp])).all(), where
            if red == "mean":
                assert np.concatenate([e.closed_count for e in ems]).tolist() == [x.n for x in exp], where
        elif dtype in FLOAT:
            assert acc.view(np.uint64).tolist() == np.array(exp, np.float64).view(np.uint64).tolist(), where
        else:
            assert acc.tolist() == exp, where

    check(ems_a, 0, "A")
    for cut in cuts:
        got = _resumed(ctx, spec, steps, snaps[cut], cut, dtype, rows=n, emit=1 << 16, cap=1000)
        _same_rows(ems_a[cut:], got, fuzzy, cut)
        check(got, cut, cut)
    return snaps, batches


def _specials(f32):
    tiny = np.float32(1e-45).item() if f32 else 5e-324
    return [np.inf, -np.inf, 0.0, -0.0, tiny, -tiny, 3 * tiny, -7 * tiny, 1.0, -1.0]


@pytest.mark.parametrize("red,dtype", [("min", "f64"), ("max", "f64"), ("min", "f32"), ("max", "f32")])
def test_float_min_max_specials(ctx, red, dtype):
    """±inf, subnormals and ±0 through the ordered-float encoding of the `acc` column: bit for bit, first of equals."""
    f32 = dtype == "f32"
    sp = np.array(_specials(f32))

    def vals(rnd, n):
        v = np.where(rnd.random(n) < 0.6, rnd.choice(sp, n), rnd.normal(0, 1e3, n))
        return v.astype(np.float32 if f32 else np.float64)

    snaps, batches = _exact_resume(ctx, red, dtype, vals, seed=10 + f32 + 2 * (red == "max"))
    # the `acc` column converts to the reference's window states: the exact min / max of each open window at the cut
    from bytewax_b200 import snapshot_rows
    from bytewax_b200.operators import windowing as win

    part = exact.fold(red, 10 * S, None, A, 3 * S, batches[:2], dtype)
    conv = snapshot_rows.window_snapshots(snaps[2], reduction=red, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=3 * S,
                                          is_float=True, classes=win)
    got = [(int(ks), w, v) for ks, sn in conv.items() for w, v in sn.logic_states.items()]
    assert len(got) > 100 and len({v for _, _, v in got}) > 5
    assert [np.float64(v).view(np.uint64) for _, _, v in got] == [np.float64(part[(k, w)]).view(np.uint64) for k, w, _ in got]


@pytest.mark.parametrize("red,dtype", [("sum", "f64"), ("sum", "f32"), ("mean", "f64"), ("mean", "f32")])
def test_float_sum_and_mean(ctx, red, dtype):
    def vals(rnd, n):
        v = rnd.normal(0, 1e3, n) * np.where(rnd.random(n) < 0.01, 1e12, 1.0)
        return v.astype(np.float32 if dtype == "f32" else np.float64)

    snaps, _ = _exact_resume(ctx, red, dtype, vals, offset=5 * S, seed=20 + (dtype == "f32") + 2 * (red == "mean"))
    if red == "mean":
        assert (snaps[2]["count"] > 0).all()  # the mean's divisor travels in the `count` column


@pytest.mark.parametrize("red,dtype", [("sum", "i64"), ("sum", "u64"), ("min", "u64"), ("max", "u64"), ("min", "i64")])
def test_integer_range(ctx, red, dtype):
    """i64 sums that wrap; u64 over its whole range (sum wraps mod 2^64, min / max unsigned)."""
    def vals(rnd, n):
        if dtype == "u64":
            return rnd.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
        v = rnd.integers(2**61, 2**63 - 1, n, dtype=np.int64)
        return np.where(rnd.random(n) < 0.5, v, -v)

    _exact_resume(ctx, red, dtype, vals, offset=5 * S, seed=30 + len(red) + len(dtype))


@pytest.mark.parametrize("red,offset", [("sum", None), ("count", 3 * S)])
def test_ordered(ctx, red, offset):
    """ordered=True with disorder inside the wait and late rows: every cut, against the C oracle."""
    spec = _spec(red, 10 * S, offset, 3 * S, ordered=True)
    rnd = np.random.default_rng(40 + (offset or 0) // S)
    batches = []
    for b in range(6):
        keys, ts = _inorder(rnd, 10_000, 400, A + b * 8 * S)
        batches.append((keys, ts + rnd.integers(-5 * S, 2 * S, len(ts)), rnd.integers(-1000, 1000, len(ts))))
    want = _coracle(spec, batches)
    assert len(want["late"][0]) > 10
    _resume_every_cut(ctx, spec, batches, want=want, rows=10_000)


# ---------------------------------------------------------------------------- 5. the path at the cut


def _expect(mode, branch):
    """(combined_folds, split_batches, slow_batches) an activation adds (as in test_gpu_late_split.py)."""
    if mode == "direct":
        return (0, 0, int(branch in ("split", "sort")))
    return {"seg": (1, 0, 0), "split": (1, 1, 0), "sort": (0, 0, 1), "wide": (0, 0, 0)}[branch]


def test_path_at_the_cut(ctx, fold_mode, monkeypatch):
    """Snapshots right after an activation on each path: the segment fold, the late split, a scatter spill (a key with
    40 % of the rows overflows its lane: 16 staging rows per bucket, as in test_gpu_stream_paths.py's hot-bucket case),
    the sort path and the direct kernel (too many panes for the segment fold).  Each path is asserted through
    `bw_stats`, the spill in spilled rows.  A snapshot taken between ingest and advance equals the one after that
    advance.  B from every cut == A == the C oracle."""
    from bytewax_b200 import gpu

    monkeypatch.setenv("BW_SC_STG", "16")  # (read when a fold is created: A and every B)
    spec = _spec("sum", S, None, 0)
    n, hk = (1 << 15) + 1023, 7
    rnd = np.random.default_rng(50)
    t0 = A + 7200 * S
    batches, branches = [], []
    for b, br in enumerate(["seg", "split", "seg", "sort", "wide", "seg"]):
        start = t0 + b * 8 * S if b < 5 else t0 + 4 * 8 * S + 150 * S
        keys, ts = _inorder(rnd, n, 100_000, start, 140 * S if br == "wide" else 8 * S)
        if b == 2:
            keys[rnd.random(n) < 0.4] = hk
        if br == "split":
            _straggle(keys, ts, _apart(rnd, n, 40))
        if br == "sort":  # more stragglers than the suspect table holds (max_batch_rows / 16)
            _straggle(keys, ts, _apart(rnd, n, n // 16 + 4000))
        batches.append((keys, ts, rnd.integers(-1000, 1000, n)))
        branches.append(br)
    want = _coracle(spec, batches)
    kw = dict(cap=1 << 17, rows=n, emit=1 << 17, late=1 << 13)
    a = gpu.WindowFold(ctx, "sum", S, None, A, 0, val_dtype="i64", capacity_hint=kw["cap"], max_batch_rows=n,
                       max_emit_rows=kw["emit"], max_late_rows=kw["late"])
    snaps, ems, prev = [a.snapshot()], [], (0, 0, 0, 0)
    try:
        for b, (keys, ts, vals) in enumerate(batches):
            a.ingest(keys, vals, ts)
            mid = a.snapshot()
            ems.append(a.advance())
            snaps.append(a.snapshot())
            _same_snapshot(mid, snaps[-1], ("between ingest and advance", b))
            st = a.stats()
            cur = (st.combined_folds, st.split_batches, st.slow_batches, st.scatter_spill_rows)
            d = tuple(c - p for c, p in zip(cur, prev))
            prev = cur
            assert d[:3] == _expect(fold_mode, branches[b]), (b, branches[b], d)
            assert (d[3] > 0) == (fold_mode == "stream" and b == 2), (b, d)  # spilled rows: the hot key's only
        ems.append(a.eof())
    finally:
        a.close()
    _check_coracle(ems, want, "A")
    steps = _batches(batches)
    for cut in range(1, len(batches) + 1):
        got = _resumed(ctx, spec, steps, snaps[cut], cut, **kw)
        _same_rows(ems[cut:], got, False, cut)


# ---------------------------------------------------------------------------- 6. gmax matters


def test_restored_gmax_makes_old_rows_late(ctx, fold_mode):
    """After the cut, one activation whose rows are in order among themselves but 12 s or more behind the restored keys'
    newest rows (wait 2 s): they are late.  Without the restored stream maximum the streaming path would take the
    activation for a clean one and fold them."""
    spec = _spec("sum", 10 * S, None, 2 * S)
    rnd = np.random.default_rng(60)
    batches = []
    for b in range(3):
        keys, ts = _inorder(rnd, 30_000, 2000, A + b * 8 * S)
        batches.append((keys, ts, rnd.integers(-100, 100, len(ts))))
    keys, ts = _inorder(rnd, 30_000, 2000, A + 2 * 8 * S - 12 * S, 4 * S)
    batches.append((keys, ts, rnd.integers(-100, 100, len(ts))))
    keys, ts = _inorder(rnd, 30_000, 2000, A + 3 * 8 * S)
    batches.append((keys, ts, rnd.integers(-100, 100, len(ts))))
    want = _coracle(spec, batches)
    assert (want["late"][4] == 3).sum() == 30_000  # every row of the activation after the cut is late
    snaps = _resume_every_cut(ctx, spec, batches, want=want, rows=30_000, late=1 << 16)
    assert snaps[3]["gmax_ts_us"] == int(batches[2][1].max())


# ---------------------------------------------------------------------------- 7. scale


def test_c1_cut_at_scale(ctx, fold_mode):
    """C1's shape at 2^20 rows per activation over 10^6 keys, cut after activation 3 of 6, restored into a table exactly
    as large as its keys need: the rows after the cut equal the C oracle's, per activation."""
    from bytewax_b200 import gpu

    n_keys, nb, B = 1_000_000, 6, 1 << 20
    L = (nb * B // 4 // 1000) * 1000
    kw = dict(val_dtype="u64", ts_from_value=True, max_batch_rows=B, max_emit_rows=1 << 22)
    a = gpu.WindowFold(ctx, "count", L, None, A, 0, capacity_hint=n_keys, **kw)
    dk, dv = ctx.dev_alloc(B * 8), ctx.dev_alloc(B * 8)
    orc = coracle.COracle("count", L, align_us=A)
    cut, got_a, got_b = 3, [], []
    try:
        for b in range(nb):
            a.gen_c1(dk, dv, b * B, B, n_keys)
            a.ingest_device(dk, dv, None, B)
            got_a.append(a.advance())
            k2, t2, _ = coracle.gen_c1(b * B, B, n_keys, A)
            orc.on_batch(k2, t2)
            if b == cut - 1:
                snap = a.snapshot()
        got_a.append(a.eof())
        orc.on_eof()
        live = len(np.unique(snap["key"]))
        assert live > 500_000
        bf = gpu.WindowFold(ctx, "count", L, None, A, 0, capacity_hint=live, **kw)
        try:
            bf.restore(snap)
            for b in range(cut, nb):
                bf.gen_c1(dk, dv, b * B, B, n_keys)
                bf.ingest_device(dk, dv, None, B)
                got_b.append(bf.advance())
            got_b.append(bf.eof())
        finally:
            bf.close()
        ck, cw, ca, _, cact = orc.closed()
        for j, em in enumerate(got_b):
            sel = cact == cut + j
            assert np.array_equal(em.closed_key, ck[sel]) and np.array_equal(em.closed_window_id, cw[sel]), j
            assert np.array_equal(em.closed_acc.astype(np.int64), ca[sel]), j
        assert sum(len(e.closed_key) for e in got_b) > 500_000
        _same_rows(got_a[cut:], got_b, False, "c1")
    finally:
        a.close()
        orc.close()
        ctx.dev_free(dk)
        ctx.dev_free(dv)


# ---------------------------------------------------------------------------- 8. capacity and API errors


@pytest.mark.parametrize("n_keys", [SEG, SEG + 1])
def test_restore_capacity(ctx, n_keys):
    """SEG keys fill a one-segment table exactly (probe chains wrap inside the segment); SEG + 1 keys do not fit it and
    restoring them fails loudly with BW_ERR_CAPACITY, and fit the smallest table that holds them (two segments)."""
    from bytewax_b200 import _native as N

    spec = _spec("sum", 10 * S, None, 2 * S)
    rnd = np.random.default_rng(70 + n_keys)
    ks = rnd.choice(np.arange(1, 10**9), n_keys, replace=False).astype(np.uint64)
    batches = []
    for b in range(3):
        keys = np.concatenate([ks, rnd.choice(ks, 2000)])
        ts = (A + b * 8 * S + (np.arange(len(keys)) * 8 * S) // len(keys)).astype(np.int64)
        batches.append((keys, ts, rnd.integers(-100, 100, len(keys))))
    steps = _batches(batches)
    kw = dict(rows=1 << 13)
    ems_a, snaps = _uninterrupted(ctx, spec, steps, cap=1 << 14, **kw)
    assert len(np.unique(snaps[1]["key"])) == n_keys
    one_seg = SEG // 2   # capacity_hint / load 0.5 = SEG slots
    if n_keys > SEG:
        b = _make(ctx, spec, cap=one_seg, **kw)
        try:
            with pytest.raises(N.BwError) as e:
                b.restore(snaps[1])
            assert e.value.status == 3 and "restore failed" in str(e.value), str(e.value)
        finally:
            b.close()
    got = _resumed(ctx, spec, steps, snaps[1], 1, cap=one_seg if n_keys <= SEG else one_seg + 1, **kw)
    _same_rows(ems_a[1:], got, False, n_keys)
    _check_coracle(ems_a, _coracle(spec, batches), "A")


def test_restore_api_errors(ctx):
    """Restore into a fold that already ingested: BW_ERR_STATE.  A snapshot after EOF: BW_ERR_STATE.  A restore with a
    column missing: BW_ERR_SPEC."""
    import ctypes as C

    from bytewax_b200 import _native as N

    spec = _spec("count", 10 * S)
    a = _make(ctx, spec)
    b = _make(ctx, spec)
    c = _make(ctx, spec)
    try:
        a.ingest(np.arange(10, dtype=np.uint64), None, np.full(10, A, np.int64))
        a.advance()
        snap = a.snapshot()
        b.ingest(np.arange(3, dtype=np.uint64), None, np.full(3, A, np.int64))
        with pytest.raises(N.BwError) as e:
            b.restore(snap)
        assert e.value.status == 5 and "freshly created" in str(e.value)
        a.eof()
        with pytest.raises(N.BwError) as e:
            a.snapshot()
        assert e.value.status == 5 and "after eof" in str(e.value)
        sn = N.BwSnapshot()
        sn.n = len(snap["key"])
        keep = []
        for name, dt in (("key", np.uint64), ("pane_id", np.int64), ("acc", np.uint64), ("count", np.uint64),
                         ("open_seq", np.uint64), ("max_ts_us", np.int64)):  # (no closed_upto)
            arr = np.ascontiguousarray(snap[name], dtype=dt)
            keep.append(arr)
            setattr(sn, name, arr.ctypes.data_as(C.POINTER(C.c_int64 if dt is np.int64 else C.c_uint64)))
        sn.batch_no, sn.gmax_ts_us, sn.last_epoch = snap["batch_no"], snap["gmax_ts_us"], snap["last_epoch"]
        with pytest.raises(N.BwError) as e:
            N.check(c.lib.bw_snapshot_load(c.h, C.byref(sn)), ctx.h)
        assert e.value.status == 4 and "missing column" in str(e.value)
    finally:
        a.close()
        b.close()
        c.close()


# ---------------------------------------------------------------------------- 9. world rescale


def _in_threads(world, fn):
    results, errors = [None] * world, [None] * world

    def main(r):
        try:
            results[r] = fn(r)
        except BaseException as ex:  # noqa: BLE001 - re-raised by the caller's thread
            errors[r] = ex

    threads = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for ex in errors:
        if ex is not None:
            raise ex
    return results


def _dest(keys, world):
    """po.dest_rank of every key."""
    u, inv = np.unique(keys, return_inverse=True)
    return np.array([po.dest_rank(int(k), world) for k in u.tolist()], dtype=np.int64)[inv]


def join_snapshots(snaps):
    """One snapshot from per-rank ones: the columns concatenated; batch_no, gmax_ts_us and last_epoch the largest."""
    out = {n: np.concatenate([s[n] for s in snaps]) for n in SNAP_COLS}
    out.update({n: max(s[n] for s in snaps) for n in ("batch_no", "gmax_ts_us", "last_epoch")})
    return out


def _world_batches(world, nb, seed):
    """Per activation, one slice per source rank."""
    rnd = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        per_rank = []
        for _ in range(world):
            ts = A + b * 12 * S + rnd.integers(-6 * S, 12 * S, 6000)
            per_rank.append(((rnd.integers(0, 3000, 6000) * 7919).astype(np.uint64), ts.astype(np.int64),
                             rnd.integers(-100, 100, 6000)))
        out.append(per_rank)
    return out


def _run_ranks(ctx, world, spec, batches, snap=None, cut_after=None):
    """Each rank of a `world` (a loopback world when world > 1) restores `snap` if given, then ingests its slices;
    returns per rank (emissions, snapshot after `cut_after` activations, snapshot right after the restore)."""
    from bytewax_b200 import gpu

    ctxs = gpu.Context.loopback_world(world) if world > 1 else [ctx]
    folds = [None] * world

    def rank_main(r):
        f = folds[r] = _make(ctxs[r], spec, rows=1 << 15, emit=1 << 18, late=1 << 18)
        restored = None
        if snap is not None:
            f.restore(snap)
            restored = f.snapshot()
        ems, cut_snap = [], None
        for b, per_rank in enumerate(batches):
            k, t, v = per_rank[r]
            f.ingest(k, v, t)
            ems.append(f.advance())
            if b + 1 == cut_after:
                cut_snap = f.snapshot()
        ems.append(f.eof())
        return ems, cut_snap, restored

    try:
        return _in_threads(world, rank_main)
    finally:
        for f in folds:  # every rank is done with its peers' memory: only now free anything
            if f is not None:
                f.close()
        if world > 1:
            for c in ctxs:
                c.close()


@pytest.mark.parametrize("w1,w2", [(1, 2), (1, 4), (2, 1), (2, 4), (4, 1), (4, 2)])
def test_world_rescale(ctx, w1, w2):
    """A world of w1 ranks runs to the cut; the per-rank snapshots are joined and every rank of a world of w2 restores
    the whole: each keeps exactly the keys the route gives it.  Its rows after the cut equal the C oracle's replay of its
    own keys, and the union over ranks equals the rows of one uninterrupted rank."""
    spec = _spec("sum", 10 * S, 5 * S, 2 * S)
    cut = 3
    pre = _world_batches(w1, cut, 80 + w1)
    post = _world_batches(w2, 3, 90 + w2)
    before = _run_ranks(ctx, w1, spec, pre, cut_after=cut)
    joined = join_snapshots([r[1] for r in before])
    after = _run_ranks(ctx, w2, spec, post, snap=joined)
    keys_all = np.unique(joined["key"])
    dest = {int(k): po.dest_rank(int(k), w2) for k in keys_all}
    flat = lambda per_rank: tuple(np.concatenate([p[i] for p in per_rank]) for i in range(3))  # noqa: E731
    for d in range(w2):
        held = set(after[d][2]["key"].tolist())
        assert held == {k for k, r in dest.items() if r == d}, d
        mine = []
        for per_rank in pre + post:
            k, t, v = flat(per_rank)
            m = _dest(k, w2) == d
            mine.append((k[m], t[m], v[m]))
        _check_coracle(after[d][0], _after(_coracle(spec, mine), cut), (w1, w2, d))
    one = _run_ranks(ctx, 1, spec, [[flat(p)] for p in pre + post])[0][0]
    rows = lambda ems: sorted(zip(*[np.concatenate([e.closed_key for e in ems]).tolist(),  # noqa: E731
                                    np.concatenate([e.closed_window_id for e in ems]).tolist(),
                                    np.concatenate([e.closed_acc for e in ems]).tolist()]))
    assert rows([e for r in after for e in r[0]]) == rows(one[cut:])
    late = lambda ems: sorted(zip(np.concatenate([e.late_key for e in ems]).tolist(),  # noqa: E731
                                  np.concatenate([e.late_window_id for e in ems]).tolist(),
                                  np.concatenate([e.late_ts_us for e in ems]).tolist()))
    assert late([e for r in after for e in r[0]]) == late(one[cut:])
    assert len(rows(one[cut:])) > 1000 and len(late(one[cut:])) > 10


# ---------------------------------------------------------------------------- 10. device columns to the reference's snapshot


def _us(d):
    from datetime import datetime, timezone

    delta = d - datetime(1970, 1, 1, tzinfo=timezone.utc)
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


NOW_US = 1_893_456_000_000_000  # 2030-01-01T00:00:00Z: the frozen system clock of the goldens


@pytest.mark.parametrize("red,length,offset,wait,ordered",
                         [c + (False,) for c in streams.SNAPSHOT_CASES] + streams.SNAPSHOT_DEVICE_CASES)
def test_device_snapshot_is_the_references(ctx, golden_dir, red, length, offset, wait, ordered):
    """The real `bw_snapshot_take` at the cut of each snapshot case, converted by `snapshot_rows.window_snapshots`:
    the same keys, windows in the same (first-opened) order with the same bounds, the same accumulators and the same
    clock difference as the reference's own `_WindowLogic.snapshot()` held."""
    from bytewax_b200 import snapshot_rows
    from bytewax_b200.operators import windowing as win

    with open(os.path.join(golden_dir, "snapshot_cases.json")) as f:
        ref = json.load(f)[streams.snapshot_case_name(red, length, offset, wait, ordered)]["keys"]
    spec, batches, cut = streams.snapshot_case(red, length, offset, wait, ordered)
    off = spec["offset_us"] or spec["length_us"]
    fold = _make(ctx, spec)
    try:
        for keys, ts, vals in batches[:cut]:
            fold.ingest(keys, vals, ts)
            fold.advance()
        snap = fold.snapshot()
    finally:
        fold.close()
    snaps = snapshot_rows.window_snapshots(snap, reduction=red, length_us=spec["length_us"], offset_us=off, align_us=A,
                                           wait_us=spec["wait_us"], now_us=NOW_US, frozen_now_us=NOW_US, ordered=ordered,
                                           classes=win)
    assert set(snaps) == set(ref)
    if (red, length, offset, wait, ordered) in streams.SNAPSHOT_DEVICE_CASES:
        assert sum(len(c["opened"]) >= 2 for c in ref.values()) >= 3
    for ks, real in ref.items():
        mine = snaps[ks]
        assert [[w, _us(m.open_time), _us(m.close_time), sorted(m.merged_ids)] for w, m in mine.windower_state.opened.items()] == real["opened"], ks
        assert dict((w, v) for w, v in real["logic_states"]) == mine.logic_states, ks
        assert _us(mine.clock_state.watermark_base) - _us(mine.clock_state.system_time_of_max_event) == real["clock_diff_us"], ks
        assert mine.queue == []
