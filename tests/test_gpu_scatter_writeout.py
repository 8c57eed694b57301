"""Edges of the bucket scatter's write-out (k_scatter, bw_stream.cuh).  Needs an H100: -m gpu.

A write-out ends every lane on a whole 32-byte sector: a bucket that has assembled an odd number of records keeps the
last one as the first staging row of its next write-out.  Rows past a bucket's staging rows wait in a block-wide
overflow area in shared memory, and only when that area is full go straight to their lane.  Each case builds its rows
tile by tile (2048 rows per tile; a block takes tiles b, b + grid, ... with one block per SM) so that chosen buckets
get chosen record counts in every write-out, and compares the closed windows with the C oracle row for row.  Every
case has a partial last tile whose row count is not a multiple of 4."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from tests.test_gpu_stream_paths import _run, _segment_of, _set  # noqa: E402

A = 1_640_995_200_000_000
TILE = 2048
STRIDE = 64  # a chosen bucket's rows sit at tile offsets slot, slot + 64, ...: at most 32 per tile, 64 such buckets


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def grid():
    """Scatter blocks: one per SM of device 0 (the lanes of a bucket), from the driver API."""
    import ctypes

    cu = ctypes.CDLL("libcuda.so.1")
    dev, sms = ctypes.c_int(), ctypes.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(ctypes.byref(sms), 16, dev) == 0  # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return sms.value


@pytest.fixture(autouse=True)
def stream_on(monkeypatch):
    monkeypatch.setenv("BW_STREAM", "1")
    for k in ("BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES", "BW_SEG_SHIFT"):
        monkeypatch.delenv(k, raising=False)


def _keys_by_segment(cap, n_cand=400_000):
    cand = np.arange(1, n_cand, dtype=np.uint64) * np.uint64(0x10001)
    return cand, _segment_of(cand, cap)


def _batches(n, grid, cap, chosen, pool_keys, seed, nb=2):
    """`chosen`: (keys, rows in a block's first tile, rows in each later tile) per bucket; those rows sit at fixed
    offsets of every tile; the other rows draw from pool_keys.  Event time from the value: 1 us per row."""
    rnd = np.random.default_rng(seed)
    tile = np.arange(n) // TILE
    off = np.arange(n) % TILE
    first = tile < grid
    out = []
    for b in range(nb):
        keys = pool_keys[rnd.integers(0, len(pool_keys), n)]
        for slot, (ck, n_first, n_later) in enumerate(chosen):
            sel = (off % STRIDE == slot) & (off // STRIDE < np.where(first, n_first, n_later))
            keys[sel] = ck[rnd.integers(0, len(ck), int(sel.sum()))]
        ts = A + b * n + np.arange(n, dtype=np.int64)
        out.append((keys, ts, (ts - A).astype(np.uint64)))
    return out


def _check(ctx, batches, hint, cap):
    st = _run(ctx, "count", 250_000, None, 0, batches, dtype="u64", capacity_hint=hint, ts_from_value=True)
    assert st.table_capacity == cap
    assert st.combined_folds == len(batches) and st.slow_batches == 0 and st.scatter_spill_rows == 0


@pytest.mark.parametrize("every", [1, 2, 3])
def test_odd_record_left_every_write_out(ctx, grid, monkeypatch, every):
    """16 staging rows per bucket.  Bucket 0 gets 7 rows in a block's first tile and 8 in every later one, bucket 1
    21 and 22: with a write-out every 1, 2 or 3 tiles both have assembled an odd number of records at every write-out.
    Bucket 0's odd record stays behind from staging, bucket 1's from the overflow area (or, when the other buckets
    have filled that area, bucket 1 writes everything)."""
    _set(monkeypatch, stg=16, every=every)
    hint, cap = 1 << 19, 1 << 20  # 256 buckets
    cand, seg = _keys_by_segment(cap)
    chosen = [(cand[seg == 0][:5], 7, 8), (cand[seg == 1][:5], 21, 22)]
    pool = cand[seg >= 2][:50_000]
    n = grid * 3 * TILE + 1023  # block 0 also gets a fourth, partial tile
    _check(ctx, _batches(n, grid, cap, chosen, pool, seed=every), hint, cap)


@pytest.mark.parametrize("stg", [12, 16])
def test_hot_buckets_overflow_every_tile(ctx, grid, monkeypatch, stg):
    """Skewed keys: one key per segment in 8 segments takes 23 rows of every tile, more than the staging rows, so those
    buckets put rows in the overflow area at every tile and keep an odd record at every write-out (one per tile)."""
    _set(monkeypatch, stg=stg, every=1)
    hint, cap = 1 << 19, 1 << 20
    cand, seg = _keys_by_segment(cap)
    chosen = [(cand[seg == 3 * i + 5][:1], 23, 23) for i in range(8)]
    pool = cand[np.isin(seg, [3 * i + 5 for i in range(8)], invert=True)][:50_000]
    n = grid * 2 * TILE + 1023
    _check(ctx, _batches(n, grid, cap, chosen, pool, seed=11 + stg), hint, cap)


def test_overflow_area_full(ctx, grid, monkeypatch):
    """More rows past their staging between two write-outs than the overflow area holds (1024 rows): 256 buckets with
    16 staging rows, written out only after a block's last tile (~24 rows per bucket: ~2000 past their staging).  The
    rows the area cannot take go straight to their lane."""
    _set(monkeypatch, stg=16, every=1000)
    hint, cap = 1 << 19, 1 << 20
    cand, _ = _keys_by_segment(cap)
    n = grid * 3 * TILE + 1023
    _check(ctx, _batches(n, grid, cap, [], cand[:50_000], seed=7), hint, cap)


def test_tile_outruns_staging(ctx, grid, monkeypatch):
    """4 buckets with 16 staging rows: every tile puts ~500 rows in each bucket, so rows go straight to their lane
    (no overflow area for such a shape) and no write-out keeps a record."""
    _set(monkeypatch, stg=16, every=1)
    hint, cap = 8192, 16384
    cand, _ = _keys_by_segment(cap)
    n = grid * 2 * TILE + 1023
    _check(ctx, _batches(n, grid, cap, [], cand[:4000], seed=3), hint, cap)


def test_c1_shape_partial_last_tile(ctx):
    """C1's own settings (10^6 keys: 489 buckets, 16 staging rows, a write-out every 3 tiles, overflow area) with a
    partial last tile of 1023 rows: n is a multiple of neither 2048 nor 4."""
    from oracle import coracle

    n = (1 << 21) + 1023
    batches = [coracle.gen_c1(b * n, n, 1_000_000, A) for b in range(2)]
    st = _run(ctx, "count", 1_000_000, None, 0, batches, dtype="u64", capacity_hint=1_000_000, ts_from_value=True)
    assert st.combined_folds == len(batches) and st.slow_batches == 0 and st.scatter_spill_rows == 0
