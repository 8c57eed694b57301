"""Branches of the streaming path that ordinary inputs never reach.  Needs an H100: -m gpu.

Each case is compared with the C oracle row for row (counts and integer sums bit for bit, float sums within the
error bound of binary64 summation against oracle/exact.py) and asserts through `bw_stats` that it took the branch it is
named for: rows in the spill list (`scatter_spill_rows`), the segment fold (`combined_folds`) or the direct kernel."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import coracle, exact  # noqa: E402  (checker only)

S = 1_000_000
A = 1_640_995_200_000_000


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def stream_on(monkeypatch):
    monkeypatch.setenv("BW_STREAM", "1")
    for k in ("BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES", "BW_SEG_SHIFT"):
        monkeypatch.delenv(k, raising=False)


def _run(ctx, red, length, offset, wait, batches, dtype="i64", capacity_hint=1 << 17, ts_from_value=False, exact_check=False,
         closes=True):
    """Fold every activation (advance after each) and replay it through the C oracle; returns the fold's stats."""
    from bytewax_b200 import gpu

    is_float = dtype == "f64"
    n = max(len(k) for k, _, _ in batches)
    fold = gpu.WindowFold(ctx, red, length, offset, A, wait, val_dtype=dtype, ts_from_value=ts_from_value,
                          capacity_hint=capacity_hint, max_batch_rows=n, max_emit_rows=1 << 22, max_late_rows=1 << 16)
    orc = coracle.COracle(red, length, offset, A, wait, False, is_float=is_float)
    ems = []
    for keys, ts, vals in batches:
        fold.ingest(keys, vals, None if ts_from_value else ts)
        orc.on_batch(keys, ts, vals)
        ems.append(fold.advance())
    ems.append(fold.eof())
    orc.on_eof()
    st = fold.stats()
    fold.close()
    ck, cw, ca, _, cact = orc.closed()
    assert orc.late()[0].size == 0
    orc.close()
    for b, e in enumerate(ems):
        sel = cact == b
        assert np.array_equal(e.closed_key, ck[sel]), (b, len(e.closed_key), int(sel.sum()))
        assert np.array_equal(e.closed_window_id, cw[sel]), b
        if not is_float:
            assert np.array_equal(e.closed_acc.astype(np.int64), ca[sel]), b
    if closes:
        assert sum(len(e.closed_key) for e in ems[:-1]) > 0  # windows closed before EOF too
    if is_float or exact_check:
        want = exact.fold(red, length, offset, A, wait, batches, dtype)
        gk = np.concatenate([e.closed_key for e in ems]).tolist()
        gw = np.concatenate([e.closed_window_id for e in ems]).tolist()
        ga = np.concatenate([e.closed_acc for e in ems])
        exp = [want[kw] for kw in zip(gk, gw)]
        if is_float:
            assert (np.abs(ga - [e.fsum for e in exp]) <= [e.bound() for e in exp]).all()
        else:
            assert ga.astype(np.int64).tolist() == exp
    return st


# ---------------------------------------------------------------------------- key skew -> spill list


def _skewed(shape, seed, nb=2, n=(1 << 20) + 1021, n_keys=100_000):
    rnd = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        ts = A + b * 4 * S + (np.arange(n) * 4 * S) // n
        if shape == "zipf":
            keys = rnd.zipf(1.1, n)
            keys = np.where(keys <= n_keys, keys - 1, rnd.integers(0, n_keys, n))
        else:
            keys = rnd.integers(0, n_keys if shape != "uniform" else 100_000, n)
            if shape != "uniform":
                keys[rnd.random(n) < 0.45] = 77  # one key carries 45 % of the rows
        if shape == "hot_sliding":  # disorder inside the wait: first-open order is not window-id order
            ts = ts + rnd.integers(-S, S + 1, n)
        out.append((keys.astype(np.uint64), ts.astype(np.int64), rnd.integers(-1000, 1000, n)))
    return out


@pytest.mark.parametrize("red,dtype", [("count", "i64"), ("sum", "i64"), ("sum", "f64")])
@pytest.mark.parametrize("shape", ["hot", "zipf", "hot_sliding", "uniform"])
def test_skewed_keys_spill(ctx, shape, red, dtype):
    """A hot key (45 % of the rows), Zipf(1.1) over 10^5 keys, and a hot key in a sliding fold with disorder inside
    `wait`: lanes overflow into the spill list, those rows are folded first by `k_spill`, and they are neither lost nor
    counted twice; the first-open order of a key whose rows are split between spill list and lane is the oracle's."""
    if shape == "uniform" and red != "count":
        pytest.skip("one uniform control is enough")
    # (the sliding hot key is kept small: its spilled rows go through the general path's per-key pane list, whose cost
    # grows with the square of that key's rows -- DESIGN.md section 10)
    batches = _skewed(shape, 21, n=(1 << 14) + 1021 if shape == "hot_sliding" else (1 << 20) + 1021)
    if dtype == "f64":
        rnd = np.random.default_rng(5)
        batches = [(k, t, rnd.normal(0, 1e3, len(k))) for k, t, _ in batches]
    sliding = shape == "hot_sliding"
    st = _run(ctx, red, 2 * S, S if sliding else None, 3 * S if sliding else 0, batches, dtype=dtype, capacity_hint=100_000)
    assert st.combined_folds == len(batches) and st.slow_batches == 0
    if shape == "uniform":
        assert st.scatter_spill_rows == 0
    else:
        assert st.scatter_spill_rows > 0


# ---------------------------------------------------------------------------- staging x segment size


def _c1(nb, n, n_keys, hot=False):
    out = []
    for b in range(nb):
        keys, ts, vals = coracle.gen_c1(b * n, n, n_keys, A)
        if hot:
            keys = keys.copy()
            keys[np.random.default_rng(b).random(n) < 0.4] = 12345
        out.append((keys, ts, vals))
    return out


N_ODD = (1 << 20) + 1023  # neither a multiple of 2048 (partial last tile) nor of 4 (rows read directly)
# pairwise over (BW_SC_STG, BW_SC_EVERY, BW_SC_STAGES, BW_SEG_SHIFT): every pair of values of any two settings occurs
STG, EVERY, STAGES, SEG = (0, 4, 6, 8, 16), (1, None, 1000), (2, 3, 4), (10, 11, 12)
MATRIX = [(STG[i], EVERY[j], STAGES[(i + j) % 3], SEG[(i + 2 * j) % 3]) for i in range(5) for j in range(3)]


def _set(monkeypatch, stg=None, every=None, stages=None, seg=None):
    for name, v in (("BW_SC_STG", stg), ("BW_SC_EVERY", every), ("BW_SC_STAGES", stages), ("BW_SEG_SHIFT", seg)):
        if v is not None:
            monkeypatch.setenv(name, str(v))


@pytest.mark.parametrize("stg,every,stages,seg", MATRIX)
def test_staging_matrix_count(ctx, monkeypatch, stg, every, stages, seg):
    """C1-shaped count fold (event time from the value) under every staging depth, write-out cadence (each tile, the
    default rule, only after the last tile), TMA stage count and segment size."""
    _set(monkeypatch, stg, every, stages, seg)
    batches = _c1(2, N_ODD, 100_000)
    st = _run(ctx, "count", 250_000, None, 0, batches, dtype="u64", ts_from_value=True)
    assert st.combined_folds == len(batches) and st.slow_batches == 0


@pytest.mark.parametrize("stages,seg", [(s, g) for s in STAGES for g in SEG])
def test_staging_matrix_sum(ctx, monkeypatch, stages, seg):
    """An i64 sum fold (values stored beside the records, no staging) under every TMA stage count and segment size."""
    _set(monkeypatch, stages=stages, seg=seg)
    rnd = np.random.default_rng(seg * 10 + stages)
    batches = [(k, t, rnd.integers(-2**40, 2**40, len(k))) for k, t, _ in _c1(2, N_ODD, 100_000)]
    st = _run(ctx, "sum", 250_000, None, 0, batches)
    assert st.combined_folds == len(batches) and st.slow_batches == 0


@pytest.mark.parametrize("every", [None, 1000])
def test_staging_with_a_hot_bucket(ctx, monkeypatch, every):
    """16 staging rows per bucket and a key with 40 % of the rows: its bucket outruns its staging rows within a tile
    (records written straight out) and overflows its lane between two write-outs (spill list)."""
    _set(monkeypatch, 16, every)
    # (small: the hot key's spilled rows span several panes and go through the general path's per-key pane list,
    # whose cost grows with the square of that key's rows -- DESIGN.md section 10)
    batches = _c1(2, (1 << 15) + 1023, 100_000, hot=True)
    st = _run(ctx, "count", 10_000, None, 0, batches, dtype="u64", ts_from_value=True)
    assert st.combined_folds == len(batches) and st.slow_batches == 0 and st.scatter_spill_rows > 0


def test_c1_shape_default_staging(ctx):
    """C1's own shape (10^6 keys: 489 buckets, 16 staging rows, a write-out every 3 tiles) at 2^22 + 1023 rows."""
    batches = _c1(2, (1 << 22) + 1023, 1_000_000)
    st = _run(ctx, "count", 1_000_000, None, 0, batches, dtype="u64", capacity_hint=1_000_000, ts_from_value=True)
    assert st.combined_folds == len(batches) and st.slow_batches == 0 and st.scatter_spill_rows == 0


# ---------------------------------------------------------------------------- a full segment


def _khash(k):  # bw_khash (bw_common.cuh)
    with np.errstate(over="ignore"):
        k = k * np.uint64(0x9E3779B97F4A7C15)
        k ^= k >> np.uint64(32)
        return k * np.uint64(0xD6E8FEB86659FD93)


def _segment_of(k, cap, seg_shift=12):  # bw_slot_of_khash >> seg_shift
    return ((_khash(k) >> np.uint64(32)) * np.uint64(cap)) >> np.uint64(32 + seg_shift)


def _keys_in_one_segment(n, cap, seg):
    cand = np.arange(1, 40 * n * (cap >> 12), dtype=np.uint64) * np.uint64(0x10001)
    sel = cand[_segment_of(cand, cap) == seg]
    assert len(sel) >= n
    return sel[:n]


def _segment_batches(keys, reps=6, seed=31):
    rnd = np.random.default_rng(seed)
    rows = np.repeat(keys, reps)
    out = []
    for b in range(2):
        k = rnd.permutation(rows)
        ts = A + b * 5 * S + (np.arange(len(k)) * 5 * S) // len(k)
        out.append((k, ts.astype(np.int64), rnd.integers(-1000, 1000, len(k))))
    return out


@pytest.mark.parametrize("mode", ["1", "0"])
@pytest.mark.parametrize("layout", ["single", "crowded"])
def test_full_segment(ctx, monkeypatch, mode, layout):
    """Load 1.0: 4096 distinct keys in one 4096-slot segment -- the whole table (capacity_hint 2048), or one segment of
    a four-segment table -- fold exactly (the probe wraps, fingerprints collide); one key more is BW_ERR_CAPACITY."""
    from bytewax_b200 import _native as N, gpu

    monkeypatch.setenv("BW_STREAM", mode)
    if layout == "single":
        hint = 2048
        keys = np.concatenate([np.array([0, 2**64 - 2], np.uint64), np.arange(1, 4095, dtype=np.uint64) * np.uint64(1_000_003)])
        extra = np.array([2**63 + 5], np.uint64)
    else:
        hint = 8192  # 16384 slots: four segments
        sel = _keys_in_one_segment(4097, 16384, 2)
        keys, extra = sel[:4096], sel[4096:]
    assert len(np.unique(keys)) == 4096
    for red in ("count", "sum"):
        st = _run(ctx, red, 2 * S, None, 0, _segment_batches(keys), capacity_hint=hint)
        assert st.table_capacity == (4096 if layout == "single" else 16384)
        assert st.combined_folds == (2 if mode == "1" else 0) and st.slow_batches == 0
    fold = gpu.WindowFold(ctx, "count", 2 * S, None, A, 0, capacity_hint=hint, max_batch_rows=1 << 16)
    k = np.concatenate([keys, extra])
    fold.ingest(k, None, np.full(len(k), A, np.int64))
    with pytest.raises(N.BwError) as e:
        fold.advance()
    assert e.value.status == 3
    fold.close()


# ---------------------------------------------------------------------------- span and pane limits


@pytest.mark.parametrize("delta,streamed", [(2**31 - 2, True), (-(2**31 - 1), True), (2**31 - 1, False), (-(2**31), False)])
def test_relative_timestamp_range(ctx, delta, streamed):
    """Records carry ts - ts(row 0) in 32 bits, INT32_MIN and INT32_MAX excluded: a row at +(2^31 - 2) or -(2^31 - 1)
    us from row 0 takes the segment fold, one at +(2^31 - 1) or -2^31 the direct kernel; rows are the oracle's."""
    rnd = np.random.default_rng(41)
    n = 40_000
    t0 = A + 3000 * S
    batches = []
    for b in range(2):
        ts = t0 + b * 4 * S + (np.arange(n) * 4 * S) // n
        keys = rnd.integers(0, 3000, n).astype(np.uint64)
        if b == 1:
            ts[n // 2] = ts[0] + delta
        batches.append((keys, ts.astype(np.int64), rnd.integers(-1000, 1000, n)))
    wait = 10**10  # every activation is clean
    for red in ("count", "sum"):
        st = _run(ctx, red, 60 * S, None, wait, batches, exact_check=True, closes=False)
        assert st.slow_batches == 0
        assert st.combined_folds == (2 if streamed else 1)


@pytest.mark.parametrize("panes,streamed", [(127, True), (128, False)])
def test_pane_span_limit(ctx, panes, streamed):
    """The segment fold takes activations that span at most 128 panes (q_hi - q_lo = 127: 64 passes of two panes)."""
    rnd = np.random.default_rng(42)
    n = 50_000
    batches = []
    for b in range(2):
        base = A + 7 * S // 10 + b * 200 * S
        ts = base + (np.arange(n) * panes * S) // (n - 1)
        # 20 keys per pane: no key holds more than one live pane (the close kernel re-ranks at most 64 per key)
        keys = (((ts - A) // S) * 20 + rnd.integers(0, 20, n)).astype(np.uint64)
        batches.append((keys, ts.astype(np.int64), rnd.integers(-1000, 1000, n)))
    assert (batches[0][1][-1] - A) // S - (batches[0][1][0] - A) // S == panes
    for red in ("count", "sum"):
        st = _run(ctx, red, S, None, 10**10, batches, exact_check=True, closes=False)
        assert st.slow_batches == 0
        assert st.combined_folds == (2 if streamed else 0)
