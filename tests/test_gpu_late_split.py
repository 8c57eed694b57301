"""The late-row split of the streaming fold (bw_late.cuh) on every branch, at its table limits and under a moving clock.
Needs an H100: -m gpu.

Every case runs three ways -- streaming with the split (the default), the sort path behind the same scatter
(BW_LATE_SPLIT=0) and the direct kernel alone (BW_STREAM=0) -- and each must equal the oracle: the C oracle for rows,
late rows (window id, value bits, timestamp) and per-activation order; oracle/exact.py for float sums and means and
for u64 / wrapping accumulators; oracle/pyoracle.py under a moving system clock.  Each case names the branch every
activation must take and asserts it through `bw_stats`, and `suspect_mask` (the exact suspect rule of
k_late_suspect) checks the preconditions of the boundary cases, so that a case cannot silently stop reaching its
branch."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import coracle, exact, pyoracle as po  # noqa: E402  (checker only)

S = 1_000_000
A = 1_640_995_200_000_000
I64_MIN = -(2**63)
UTC_MIN = -62_135_596_800_000_000  # BW_UTC_MIN_US_DEV
PROBE_MAX = 4096                   # BW_LATE_PROBE_MAX
SQ = 128                           # BW_LATE_SQ
MODES = ("split", "sort", "direct")
FLOAT = ("f32", "f64")


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


# ---------------------------------------------------------------------------- the rules the tests reason with


def suspect_mask(ts, gprev, wait):
    """Rows k_late_suspect must find: ts_i < wm(max(gprev, ts_0 .. ts_{i-1})), wm(m) = max(UTC_MIN, m - wait) with
    wm(INT64_MIN) = UTC_MIN (bw_wm_of).  `gprev`: the largest timestamp of the earlier activations."""
    ts = np.asarray(ts, np.int64)
    prev = np.empty_like(ts)
    prev[0] = gprev
    prev[1:] = ts[:-1]
    pm = np.maximum.accumulate(prev)
    with np.errstate(over="ignore"):
        wm = np.maximum(pm - np.int64(wait), np.int64(UTC_MIN))
    wm[pm < I64_MIN + wait] = UTC_MIN  # (bw_sub_sat saturates at INT64_MIN)
    if wait == 0:
        wm[pm == I64_MIN] = UTC_MIN
    return ts < wm


def suspect_masks(batches, wait):
    out, gprev = [], I64_MIN
    for _, ts, _ in batches:
        out.append(suspect_mask(ts, gprev, wait))
        gprev = max(gprev, int(np.max(ts)))
    return out


def late_masks(batches, wait):
    """Late rows of a frozen clock: ts < (the largest earlier timestamp of the row's key) - wait.  (No key is ever
    discarded with a frozen clock: a row opens a window that closes after its own watermark.)"""
    mx, out = {}, []
    for keys, ts, _ in batches:
        m = np.zeros(len(keys), bool)
        for i, (k, t) in enumerate(zip(keys.tolist(), ts.tolist())):
            cur = mx.get(k)
            if cur is not None and t < max(cur - wait, UTC_MIN):
                m[i] = True
            elif cur is None or t > cur:
                mx[k] = t
        out.append(m)
    return out


# ---------------------------------------------------------------------------- inputs


def _inorder(rnd, n, n_keys, t0, span=8 * S):
    keys = rnd.integers(0, n_keys, n).astype(np.uint64)
    ts = (t0 + (np.arange(n) * span) // n).astype(np.int64)
    return keys, ts


def _straggle(keys, ts, at, back=40 * S):
    """Rows `at` (>= 1) become stragglers: the key of the row before, `back` behind its timestamp."""
    at = np.asarray(at)
    keys[at] = keys[at - 1]
    ts[at] = ts[at - 1] - back


def _apart(rnd, n, k):
    """k row indices in 2 .. n - 1, no two adjacent (a straggler's key is then always that of an on-time row)."""
    return np.sort(rnd.choice(np.arange(2, n, 2), k, replace=False))


def _vals(rnd, n, dtype="i64"):
    if dtype == "f64":
        return rnd.normal(0, 1e3, n)
    if dtype == "f32":
        return rnd.normal(0, 1e3, n).astype(np.float32)
    if dtype == "u64":
        return rnd.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    return rnd.integers(-1000, 1000, n)


# ---------------------------------------------------------------------------- fold three ways, check against the oracle


def _oracle_vals(vals, dtype):
    return np.asarray(vals).astype(np.float64) if dtype in FLOAT else np.asarray(vals).view(np.int64)


def _oracle(batches, red, length, offset, wait, dtype, ordered, exact_acc):
    """Rows and late rows from the C oracle (fed `count` when the accumulators come from oracle/exact.py)."""
    orc = coracle.COracle("count" if exact_acc else red, length, offset, A, wait, ordered, is_float=dtype in FLOAT)
    for keys, ts, vals in batches:
        orc.on_batch(keys, ts, _oracle_vals(vals, dtype))
    orc.on_eof()
    want = dict(closed=orc.closed(), late=orc.late())
    orc.close()
    if exact_acc:
        lm = late_masks(batches, wait)
        off = offset or length
        n_late = sum(len(exact.window_ids(int(t), length, off, A)) for (_, ts, _), m in zip(batches, lm) for t in ts[m])
        assert n_late == len(want["late"][0])  # (the helper's late rows are the oracle's)
        clean = [(k[~m], t[~m], v[~m]) for (k, t, v), m in zip(batches, lm)]
        want["exact"] = exact.fold(red, length, offset, A, wait, clean, dtype)
    return want


def _check(ems, want, red, dtype, where):
    ck, cw, ca, _, cact = want["closed"]
    lk, lw, lv, lts, lact = want["late"]
    for b, e in enumerate(ems):
        sel = cact == b
        assert np.array_equal(e.closed_key, ck[sel]) and np.array_equal(e.closed_window_id, cw[sel]), (where, b)
        if "exact" not in want:
            assert np.array_equal(e.closed_acc.astype(np.int64), ca[sel]), (where, b)
        sel = lact == b
        assert np.array_equal(e.late_key, lk[sel]) and np.array_equal(e.late_window_id, lw[sel]), (where, b)
        assert np.array_equal(e.late_ts_us, lts[sel]), (where, b)
        assert np.array_equal(e.late_val.view(np.uint64), lv[sel].view(np.uint64)), (where, b)
    if "exact" in want:
        got_k = np.concatenate([e.closed_key for e in ems]).tolist()
        got_w = np.concatenate([e.closed_window_id for e in ems]).tolist()
        acc = np.concatenate([e.closed_acc for e in ems])
        exp = [want["exact"][kw] for kw in zip(got_k, got_w)]
        assert len(exp) == len(want["exact"]), where
        if red == "mean" or (red == "sum" and dtype in FLOAT):
            fs = np.array([x.fsum for x in exp])
            bound = np.array([x.bound() for x in exp])
            assert (np.abs(acc - fs) <= bound).all(), where
            if red == "mean":
                assert np.concatenate([e.closed_count for e in ems]).tolist() == [x.n for x in exp], where
        elif dtype in FLOAT:
            assert np.array_equal(acc.view(np.uint64), np.array(exp, np.float64).view(np.uint64)), where
        else:
            assert acc.tolist() == exp, where


def _fold(ctx, monkeypatch, mode, batches, red, length, offset, wait, dtype="i64", ordered=False, ts_from_value=False,
          capacity_hint=1 << 14, max_batch_rows=None, max_emit_rows=1 << 21, max_late_rows=1 << 20):
    """Every activation ingested and advanced; the rows of each advance + EOF, and what each activation added to
    (combined_folds, split_batches, slow_batches, scatter_spill_rows)."""
    from bytewax_b200 import gpu

    _set_mode(monkeypatch, mode)
    fold = gpu.WindowFold(ctx, red, length, offset, A, wait, val_dtype=dtype, ts_from_value=ts_from_value, ordered=ordered,
                          capacity_hint=capacity_hint, max_batch_rows=max_batch_rows or max(len(k) for k, _, _ in batches),
                          max_emit_rows=max_emit_rows, max_late_rows=max_late_rows)
    ems, deltas, prev = [], [], (0, 0, 0, 0)
    try:
        for keys, ts, vals in batches:
            fold.ingest(keys, vals, None if ts_from_value else ts)
            ems.append(fold.advance())
            st = fold.stats()
            cur = (st.combined_folds, st.split_batches, st.slow_batches, st.scatter_spill_rows)
            deltas.append(tuple(c - p for c, p in zip(cur, prev)))
            prev = cur
        ems.append(fold.eof())
    finally:
        fold.close()
    return ems, deltas


def _expect(mode, branch):
    """(combined_folds, split_batches, slow_batches) an activation adds.  Branches: `seg` (clean: segment fold),
    `wide` (clean, too many panes: direct kernel), `split` (late rows split off, the rest on the segment fold), `sort`
    (not clean, and the split gave up or is off: the sort path, nothing emitted by k_late_emit)."""
    if mode == "direct":
        return (0, 0, int(branch in ("split", "sort")))
    if mode == "sort":
        return {"seg": (1, 0, 0), "wide": (0, 0, 0)}.get(branch, (0, 0, 1))
    return {"seg": (1, 0, 0), "split": (1, 1, 0), "sort": (0, 0, 1), "wide": (0, 0, 0)}[branch]


def _three_ways(ctx, monkeypatch, batches, branches, red="sum", length=10 * S, offset=None, wait=0, dtype="i64",
                ordered=False, ts_from_value=False, exact_acc=None, **kw):
    """The case through all three modes; every activation's rows and branch.  Returns the split mode's deltas."""
    assert len(branches) == len(batches)
    if exact_acc is None:
        exact_acc = red == "mean" or dtype in ("u64", "f32", "f64")
    oracle_batches = batches
    if ts_from_value:
        oracle_batches = [(k, A + np.asarray(v).view(np.int64), v) for k, _, v in batches]
    want = _oracle(oracle_batches, red, length, offset, wait, dtype, ordered, exact_acc)
    out = {}
    for mode in MODES:
        ems, deltas = _fold(ctx, monkeypatch, mode, batches, red, length, offset, wait, dtype, ordered, ts_from_value, **kw)
        _check(ems, want, red, dtype, mode)
        for b, (d, br) in enumerate(zip(deltas, branches)):
            assert d[:3] == _expect(mode, br), (mode, b, br, d)
        out[mode] = deltas
    return out["split"], want


# ---------------------------------------------------------------------------- 1. suspect-table capacity


@pytest.mark.parametrize("rows,extra", [(1 << 16, 0), (1 << 16, 1), (1 << 12, 0), (1 << 12, 1)])
def test_suspect_table_capacity(ctx, monkeypatch, rows, extra):
    """L.cap = max(1024, max_batch_rows / 16) suspects take the split; one more takes the sort path."""
    cap = max(1024, rows // 16)
    ns = cap + extra
    rnd = np.random.default_rng(100 + rows + extra)
    n_keys = rows // 20
    batches = []
    for b in range(3):
        keys, ts = _inorder(rnd, rows, n_keys, A + b * 8 * S)
        if b == 1:
            _straggle(keys, ts, _apart(rnd, rows, ns))
        batches.append((keys, ts, _vals(rnd, rows)))
    assert [int(m.sum()) for m in suspect_masks(batches, 0)] == [0, ns, 0]
    _three_ways(ctx, monkeypatch, batches, ["seg", "sort" if extra else "split", "seg"], max_batch_rows=rows)


# ---------------------------------------------------------------------------- 2. a hot key in the suspect table


@pytest.mark.parametrize("hot,heavy,branch", [(2000, False, "split"), (6000, False, "sort"), (2000, True, "split")])
def test_hot_key_suspects(ctx, monkeypatch, hot, heavy, branch):
    """One key's suspects share one probe chain: ~2000 of them stay on the split, ~6000 (more than
    BW_LATE_PROBE_MAX) exhaust the probe and take the sort path.  `heavy`: the key also carries 45 % of the rows, so
    its lane overflows into the spill list in the same activation as the split."""
    rows, hk = 1 << 18, 7
    rnd = np.random.default_rng(200 + hot + heavy)
    batches = []
    for b in range(3):
        keys, ts = _inorder(rnd, rows, 100_000, A + b * 8 * S)
        if heavy:
            keys[rnd.random(rows) < 0.45] = hk
        keys[0] = hk
        if b == 1:
            at = np.sort(rnd.choice(np.arange(1, rows), hot, replace=False))
            keys[at] = hk
            ts[at] -= 40 * S
        batches.append((keys, ts, _vals(rnd, rows)))
    sus = suspect_masks(batches, 0)
    assert [int(m.sum()) for m in sus] == [0, hot, 0]
    assert (batches[1][0][sus[1]] == hk).all() and (hot > PROBE_MAX) == (branch == "sort")
    split, _ = _three_ways(ctx, monkeypatch, batches, ["seg", branch, "seg"], capacity_hint=1 << 17)
    if heavy:
        assert split[1][3] > 0  # rows spilled in the activation that was split


# ---------------------------------------------------------------------------- 3. a suspect that keeps a span past 2^31 us


@pytest.mark.parametrize("kind,branch", [("new_key", "sort"), ("late_key", "split")])
def test_row_an_hour_behind(ctx, monkeypatch, kind, branch):
    """A row an hour behind the stream in an otherwise straggling activation.  A new key's first row is a suspect
    but not late: it stays, the rows left span more than 2^31 us, the second scatter flags the range and the sort
    path takes the activation.  The same row for a key seen just before is late: it leaves, and the relative
    timestamps of the rest are counted from the newest row, so the split holds."""
    n = 60_000
    rnd = np.random.default_rng(300 + len(kind))
    batches = []
    for b in range(3):
        keys, ts = _inorder(rnd, n, 3000, A + 7200 * S + b * 8 * S)
        if b == 1:
            _straggle(keys, ts, _apart(rnd, n, 40))
            at = n // 2
            keys[at] = 10**12 if kind == "new_key" else keys[at - 1]
            ts[at] = ts[at - 1] - 3600 * S
        batches.append((keys, ts, _vals(rnd, n)))
    late = late_masks(batches, 0)[1]
    assert late[n // 2] == (kind == "late_key") and suspect_masks(batches, 0)[1][n // 2]
    _three_ways(ctx, monkeypatch, batches, ["seg", branch, "seg"])


# ---------------------------------------------------------------------------- 4. split, but too many panes


def test_split_but_too_wide(ctx, monkeypatch):
    """Tumbling 1 s windows, activations spanning 200 s: the split succeeds, what is left spans more than 128 panes,
    the sort path takes the activation and every late row is emitted exactly once."""
    n = 50_000
    rnd = np.random.default_rng(400)
    batches = []
    for b in range(3):
        ts = (A + 7 * S // 10 + b * 200 * S + (np.arange(n) * 200 * S) // n).astype(np.int64)
        keys = (((ts - A) // S) * 20 + rnd.integers(0, 20, n)).astype(np.uint64)  # (one live pane per key)
        if b == 1:
            _straggle(keys, ts, _apart(rnd, n, 30), back=5 * S)
        batches.append((keys, ts, _vals(rnd, n)))
    assert int(late_masks(batches, 0)[1].sum()) == 30
    _three_ways(ctx, monkeypatch, batches, ["wide", "sort", "wide"], length=S)


# ---------------------------------------------------------------------------- 5. every row late


def test_every_row_late(ctx, monkeypatch):
    """An activation of 1000 rows, each behind its key's watermark: the second scatter has no row at all.  Then an
    activation of a single late row."""
    rnd = np.random.default_rng(500)
    t0 = A + 100 * S
    keys = (np.arange(1000) % 50).astype(np.uint64)
    batches = [
        (keys.copy(), (t0 + np.arange(1000) * 8000).astype(np.int64), _vals(rnd, 1000)),
        (keys.copy(), (t0 - 30 * S + rnd.integers(0, 20 * S, 1000)).astype(np.int64), _vals(rnd, 1000)),
        (np.array([3], np.uint64), np.array([t0 - 5 * S], np.int64), np.array([77])),
        (keys.copy(), (t0 + 8 * S + np.arange(1000) * 8000).astype(np.int64), _vals(rnd, 1000)),
    ]
    assert [int(m.sum()) for m in suspect_masks(batches, 2 * S)] == [0, 1000, 1, 0]
    assert [int(m.sum()) for m in late_masks(batches, 2 * S)] == [0, 1000, 1, 0]
    _three_ways(ctx, monkeypatch, batches, ["seg", "split", "split", "seg"], wait=2 * S, max_batch_rows=1024)


# ---------------------------------------------------------------------------- 6. chunk and tile edges


@pytest.mark.parametrize("n", [(1 << 16) - 1, (1 << 16) - 63, 40_037])
def test_chunk_and_tile_edges(ctx, monkeypatch, n):
    """Activations whose last 64-row chunk and last 2048-row tile are partial, with suspects in row 0 (behind the
    previous activation only), the first and last rows of tiles, both rows of lane 0 and lane 31 of a chunk, and the
    activation's last two rows."""
    rnd = np.random.default_rng(600 + n)
    pos = {1, 2, 62, 63, 2048, 2049, 2048 + 62, 2048 + 63, 3 * 2048 - 1, 6 * 2048, 64 * 100 + 1, 64 * 100 + 62, n - 2, n - 1}
    pos = np.array(sorted(pos))
    batches = []
    for b in range(3):
        keys, ts = _inorder(rnd, n, 3000, A + b * 8 * S)
        if b == 1:
            keys[0] = batches[0][0][-1]
            ts[0] = batches[0][1][-1] - 40 * S
            _straggle(keys, ts, pos)
        batches.append((keys, ts, _vals(rnd, n)))
    sus = suspect_masks(batches, 0)
    assert np.flatnonzero(sus[1]).tolist() == [0] + pos.tolist() and not sus[0].any() and not sus[2].any()
    assert late_masks(batches, 0)[1][[0, n - 1]].all()
    _three_ways(ctx, monkeypatch, batches, ["seg", "split", "seg"], max_batch_rows=1 << 16)


# ---------------------------------------------------------------------------- 7. dense suspects: the direct branch


def _sm_count():
    """Multiprocessors of device 0, from the driver (CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT)."""
    import ctypes as C

    cu = C.CDLL("libcuda.so.1")
    dev, n = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0
    return n.value


def test_dense_suspects_direct_branch(ctx, monkeypatch):
    """k_late_suspect runs nw = 8 x 8 x SM count warps; in step s warp w scans chunks w + (4 s + u) nw, u = 0 .. 3.
    Warp 5 queues 50 suspects in its first step and meets 3 x 60 in its second: more than BW_LATE_SQ, so it flushes
    its queue and writes the 180 straight to the list, behind its own 50.  Warp 9 queues 100 in its first step and 100
    more in its second (the queue is flushed in the middle of the step)."""
    nw = 8 * 8 * _sm_count()
    n = 64 * (6 * nw + 64)
    rnd = np.random.default_rng(700)
    k0, t0 = _inorder(rnd, 100_000, 50_000, A)
    keys, ts = _inorder(rnd, n, 50_000, A + 8 * S)
    for w, runs in {5: ((0, 50), (4, 60), (5, 60), (6, 60)), 9: ((0, 50), (1, 50), (4, 50), (5, 50))}.items():
        for u, m in runs:
            c = 64 * (w + u * nw)
            keys[c + 64 - m: c + 64] = keys[c]
            ts[c + 64 - m: c + 64] = ts[c] - 40 * S - rnd.integers(0, S, m)
    batches = [(k0, t0, _vals(rnd, len(k0))), (keys, ts, _vals(rnd, n))]
    sus = suspect_masks(batches, 0)[1]
    by_chunk = sus[: n // 64 * 64].reshape(-1, 64).sum(axis=1)
    step = lambda w, s: int(sum(by_chunk[c] for c in w + (4 * s + np.arange(4)) * nw if c < len(by_chunk)))  # noqa: E731
    assert step(5, 0) == 50 and step(5, 1) == 180 > SQ
    assert step(9, 0) == 100 <= SQ < step(9, 0) + step(9, 1)
    assert int(sus.sum()) == 430
    _three_ways(ctx, monkeypatch, batches, ["seg", "split"], max_batch_rows=1 << 22, capacity_hint=1 << 16,
                max_emit_rows=1 << 22)


# ---------------------------------------------------------------------------- 8. the C1 shape at 2^22 rows


def test_c1_shape_with_stragglers(ctx, monkeypatch):
    """C1 (event time from a u64 value, count, wait 0) at 2^22 rows per activation -- 2048 tiles, so k_late_gpre
    scans two tiles per thread -- with 1 % of the rows sent 120 s back.  Every activation takes the split."""
    n, nb = 1 << 22, 4
    batches = []
    for b in range(nb):
        keys, _, vals = coracle.gen_c1(200 * S + b * n, n, 1_000_000, A)
        vals = vals.copy()
        back = np.random.default_rng(800 + b).random(n) < 0.01
        back[0] = False
        vals[back] -= np.uint64(120 * S)
        batches.append((keys, None, vals))
    _, want = _three_ways(ctx, monkeypatch, batches, ["split"] * nb, red="count", length=S, dtype="u64",
                          ts_from_value=True, exact_acc=False, capacity_hint=1 << 20, max_emit_rows=1 << 23,
                          max_late_rows=1 << 17)
    assert len(want["late"][0]) > 10_000


# ---------------------------------------------------------------------------- 9. suspect and late boundaries


def test_suspect_and_late_boundaries(ctx, monkeypatch):
    """wait 2 s.  In the second activation:
    row 0       key K5 at T+4 s: late only through the previous activation's maximum (K5's own at T+7 s);
    K1 at T+3 s: exactly its key's watermark (T+5 - 2): on time;  K2 at T+3 s - 1 us: late;
    K3 at T+2 s: behind the running maximum but not behind its key (T+1): a suspect, not late;
    K4 at T+2 s, and later K4 at T+7 s: the newer row arrives after it, so it stays on time;
    keys 0 and 2^64 - 1 late;
    K7 jumps 2.5 s ahead and its next row, 6 rows later in the same 64-row chunk, is late only because of that jump."""
    T, n = A + 100 * S, 5000
    K1, K2, K3, K4, K5, K7 = 10**9 + 1, 10**9 + 2, 10**9 + 3, 10**9 + 4, 10**9 + 5, 10**9 + 7
    KMAX = 2**64 - 1
    rnd = np.random.default_rng(900)

    def fill(t0):  # (filler keys 1 .. 500)
        k, t = _inorder(rnd, n, 500, t0)
        return k + np.uint64(1), t

    k0, t0 = fill(T)
    sk = np.array([K1, K2, K3, K4, K5, 0, KMAX], np.uint64)
    st = np.array([T + 5 * S, T + 5 * S, T + 1 * S, T + 1 * S, T + 7 * S, T + 6 * S, T + 6 * S], np.int64)
    k0, t0 = np.concatenate([k0, sk]), np.concatenate([t0, st])
    o = np.argsort(t0, kind="stable")
    k0, t0 = k0[o], t0[o]
    k1, t1 = fill(T + 8 * S)
    jump = 64 * 70 + 10
    place = {0: (K5, T + 4 * S), 1000: (K1, T + 3 * S), 1001: (K2, T + 3 * S - 1), 1500: (K3, T + 2 * S),
             2000: (K4, T + 2 * S), 3000: (K4, T + 7 * S), 2500: (0, T + 1 * S), 2600: (KMAX, T + 1 * S),
             jump: (K7, int(t1[jump]) + 5 * S // 2), jump + 6: (K7, int(t1[jump + 6]))}
    for i, (k, t) in place.items():
        k1[i], t1[i] = k, t
    k2, t2 = fill(T + 16 * S)
    batches = [(k0, t0, _vals(rnd, len(k0))), (k1, t1, _vals(rnd, n)), (k2, t2, _vals(rnd, n))]
    wait = 2 * S
    sus = suspect_masks(batches, wait)
    assert not sus[0].any() and not sus[2].any()
    assert sus[1][[0, 1000, 1001, 1500, 2000, 3000, 2500, 2600, jump + 6]].all() and sus[1].sum() < 1024
    # (the K7 row is a suspect only through the rows before it in its own chunk)
    before_chunk = max(int(t0.max()), int(t1[: jump // 64 * 64].max()))
    assert t1[jump + 6] >= before_chunk - wait
    late = late_masks(batches, wait)[1]
    assert sorted(int(k) for k in k1[late]) == sorted([K2, K5, 0, KMAX, K7])
    _three_ways(ctx, monkeypatch, batches, ["seg", "split", "seg"], wait=wait, max_batch_rows=1 << 13)


# ---------------------------------------------------------------------------- 10. modes and value types


@pytest.mark.parametrize("red,dtype,length,offset,ordered,kind", [
    ("count", "i64", 10, 3, True, None),    # ordered, sliding, indivisible offset
    ("mean", "f64", 10, None, False, None),
    ("sum", "f32", 10, None, False, None),
    ("min", "f32", 10, 5, False, None),
    ("max", "u64", 10, None, False, None),
    ("sum", "i64", 10, 5, False, "wrap"),   # sums wrap past 2^63
])
def test_modes_and_types_through_the_split(ctx, monkeypatch, red, dtype, length, offset, ordered, kind):
    """Stragglers with edge values in the second and third activations, every mode and value type; late rows keep
    their value bits (f32 widened to f64)."""
    rnd = np.random.default_rng(1000 + len(red) * 7 + len(dtype) + (offset or 0))
    n = 50_000
    batches = []
    for b in range(3):
        keys, ts = _inorder(rnd, n, 2000, A - 3 * S + b * 8 * S)
        if kind == "wrap":
            v = rnd.integers(2**61, 2**63 - 1, n) * rnd.choice([-1, 1], n)
        else:
            v = _vals(rnd, n, dtype)
        if b > 0:
            at = _apart(rnd, n, 60)
            _straggle(keys, ts, at)
            if dtype == "f32":
                v[at] = rnd.choice(np.array([np.finfo(np.float32).max, -np.inf, -0.0, 1e-45], np.float32), len(at))
            elif dtype == "u64":
                v[at] = rnd.choice(np.array([2**64 - 1, 2**63, 0], np.uint64), len(at))
        batches.append((keys, ts, v))
    _three_ways(ctx, monkeypatch, batches, ["seg", "split", "split"], red=red, length=length * S,
                offset=offset * S if offset else None, wait=S, dtype=dtype, ordered=ordered,
                exact_acc=None if kind is None else True)


# ---------------------------------------------------------------------------- 11. a moving system clock


def _clock_steps(seed):
    """8 activations of 20,000 rows over 2000 keys in the second before system time `now`, 0.5 % of them 30 s back, and two
    notify phases.  Key Z: an on-time row in activation 3, then, 14 s of system time later, a single row 1 s newer
    than that -- late only because its watermark drifted.  Key D: a row in activation 1, discarded by the notify
    phase at +16 s (all its windows closed), back in activation 2 with a timestamp older than that row."""
    rnd = np.random.default_rng(seed)
    now0 = A + 100 * S + 300_000
    Z, D = 10**9 + 1, 10**9 + 2
    plan = [("b", 0), ("b", 3), ("n", 16), ("b", 17), ("b", 20), ("b", 34), ("b", 37), ("n", 47), ("b", 48), ("b", 51)]
    steps, vid = [], 0
    for kind, t in plan:
        now = now0 + t * S
        if kind == "n":
            steps.append(("notify", now))
            continue
        n = 20_000
        keys = rnd.integers(0, 2000, n).astype(np.uint64)
        ts = (now - S + (np.arange(n) * S) // n).astype(np.int64)  # (the last second: only the stragglers are suspects)
        back = rnd.random(n) < 0.005
        ts[back] -= 30 * S
        if t == 3:
            keys[n // 2], ts[n // 2] = D, now - 1 * S
        if t == 17:
            keys[n // 2], ts[n // 2] = D, now0 - 2 * S
        if t == 20:
            keys[n // 2], ts[n // 2] = Z, now - 1 * S
        if t == 34:
            keys[n // 2], ts[n // 2] = Z, now0 + 20 * S
        vals = np.arange(vid, vid + n)
        vid += n
        steps.append(("batch", now, keys, ts, vals))
    return steps, Z, D


@pytest.mark.parametrize("length,offset", [(10, None), (10, 5)])
def test_moving_clock_through_the_split(ctx, monkeypatch, length, offset):
    """`set_system_now` between activations and notify phases: every activation is split in the frame where system
    time is 0.  A key whose only row of an activation is late after its watermark drifted closes its windows in that
    activation (the reference's on_batch does); a discarded key comes back with an old timestamp and is not late;
    late rows carry their absolute timestamps."""
    from bytewax_b200 import gpu

    wait = 2 * S
    steps, Z, D = _clock_steps(1100 + (offset or 0))
    spec = po.FoldSpec("sum", length * S, offset * S if offset else None, A, wait, False, now_us=steps[0][1])
    eng = po.StatefulBatchEngine(spec)
    want = []
    for s in steps:
        if s[0] == "batch":
            eng.set_now(s[1])
            want.append(eng.on_batch(s[2].tolist(), s[3].tolist(), s[4].tolist()))
        else:
            want.append(eng.on_notify(s[1]))
    want.append(eng.on_eof())
    ts_of = {int(v): int(t) for s in steps if s[0] == "batch" for v, t in zip(s[4], s[3])}
    # preconditions: Z's single row at +34 s is late and its window closes in the same activation; D's row at +17 s
    # is older than its row at +3 s less the wait, and not late
    iz = [i for i, s in enumerate(steps) if s[0] == "batch" and s[1] == steps[0][1] + 34 * S][0]
    tags = [r[2] for r in want[iz] if r[0] == Z]
    assert tags[0] == "L" and "E" in tags
    idd = [i for i, s in enumerate(steps) if s[0] == "batch" and s[1] == steps[0][1] + 17 * S][0]
    assert not [r for r in want[idd] if r[0] == D and r[2] == "L"]
    assert sum(1 for a in want for r in a if r[2] == "L") > 300
    for mode in MODES:
        _set_mode(monkeypatch, mode)
        fold = gpu.WindowFold(ctx, "sum", length * S, offset * S if offset else None, A, wait, val_dtype="i64",
                              capacity_hint=1 << 13, max_batch_rows=1 << 15, max_emit_rows=1 << 20, max_late_rows=1 << 18)
        prev = (0, 0, 0)
        try:
            for i, s in enumerate(steps + [("eof",)]):
                if s[0] == "batch":
                    fold.set_system_now(s[1])
                    fold.ingest(s[2], s[4], s[3])
                    em = fold.advance()
                    st = fold.stats()
                    cur = (st.combined_folds, st.split_batches, st.slow_batches)
                    d = tuple(c - p for c, p in zip(cur, prev))
                    prev = cur
                    assert d == {"split": (1, 1, 0), "sort": (0, 0, 1), "direct": (0, 0, 1)}[mode], (mode, i, d)
                elif s[0] == "notify":
                    em = fold.advance(system_now_us=s[1])
                else:
                    em = fold.eof()
                got_e = [(k, w, a) for k, (w, a) in em.down()]
                assert got_e == [(k, w, p) for k, w, t, p in want[i] if t == "E"], (mode, i)
                assert [(k, w, v) for k, (w, v) in em.late()] == [(k, w, p) for k, w, t, p in want[i] if t == "L"], (mode, i)
                assert em.late_ts_us.tolist() == [ts_of[int(v)] for v in em.late_val], (mode, i)
        finally:
            fold.close()


# ---------------------------------------------------------------------------- 12. the late buffer


@pytest.mark.parametrize("mode", ["split", "sort"])
def test_late_buffer_exactly_full(ctx, monkeypatch, mode):
    """`max_late_rows` equal to the late rows of the activation: it passes on the split and on the sort path; one
    row less is BW_ERR_CAPACITY on both."""
    from bytewax_b200 import _native as N

    rnd = np.random.default_rng(1200)
    n = 30_000
    batches = []
    for b in range(2):
        keys, ts = _inorder(rnd, n, 1000, A + b * 8 * S)
        if b == 1:
            _straggle(keys, ts, _apart(rnd, n, 150))
        batches.append((keys, ts, _vals(rnd, n)))
    want = _oracle(batches, "sum", 10 * S, None, 0, "i64", False, False)
    n_late = len(want["late"][0])
    assert n_late >= 140 and (want["late"][4] == 1).all()
    ems, deltas = _fold(ctx, monkeypatch, mode, batches, "sum", 10 * S, None, 0, max_late_rows=n_late)
    _check(ems, want, "sum", "i64", mode)
    assert deltas[1][:3] == _expect(mode, "split")
    with pytest.raises(N.BwError) as e:
        _fold(ctx, monkeypatch, mode, batches, "sum", 10 * S, None, 0, max_late_rows=n_late - 1)
    assert e.value.status == 3
