"""The dense key column (Table::keys) beside the hot slots equals hot[].key for every slot, after every path that claims
a slot: the segment fold's merge, the direct kernel, the scatter's spill list (k_spill), the late split, the sort path,
restore from a snapshot and the multi-rank merge of a loopback world.  Needs an H100: -m gpu."""

import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 1_640_995_200_000_000
S = 1_000_000


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def defaults(monkeypatch):
    for k in ("BW_STREAM", "BW_LATE_SPLIT", "BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES", "BW_SEG_SHIFT"):
        monkeypatch.delenv(k, raising=False)


def _batches(nb=3, n=1 << 18, n_keys=50_000, seed=7, hot_key=None, late_every=0):
    rnd = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        keys = rnd.integers(0, n_keys, n).astype(np.uint64) * np.uint64(0x9E3779B1)
        if hot_key is not None:
            keys[rnd.random(n) < 0.45] = hot_key
        ts = A + b * 4 * S + (np.arange(n) * 4 * S) // n
        if late_every and b > 0:
            ts[n // 2::late_every] -= 20 * S  # a few rows far behind the stream: late
        out.append((keys, ts.astype(np.int64), rnd.integers(-1000, 1000, n).astype(np.int64)))
    return out


def _fold(ctx, red="sum", wait=0, capacity_hint=1 << 17, n=1 << 18):
    from bytewax_b200 import gpu

    return gpu.WindowFold(ctx, red, 2 * S, None, A, wait, val_dtype="i64", capacity_hint=capacity_hint, max_batch_rows=n,
                          max_emit_rows=1 << 22, max_late_rows=1 << 18)


def _check(fold, seen):
    bad, used = fold.check_key_column()
    assert bad == 0
    assert used == len(seen)


def _run(fold, batches):
    seen = set()
    for keys, ts, vals in batches:
        fold.ingest(keys, vals, ts)
        seen.update(keys.tolist())
        _check(fold, seen)
        fold.advance()
        _check(fold, seen)
    st = fold.stats()
    fold.eof()
    _check(fold, seen)
    return st


@pytest.mark.parametrize("red", ["count", "sum", "mean"])
def test_streamed(ctx, red):
    fold = _fold(ctx, red)
    try:
        st = _run(fold, _batches())
    finally:
        fold.close()
    assert st.combined_folds == 3 and st.scatter_spill_rows == 0


def test_direct_path(ctx, monkeypatch):
    monkeypatch.setenv("BW_STREAM", "0")
    fold = _fold(ctx)
    try:
        st = _run(fold, _batches())
    finally:
        fold.close()
    assert st.combined_folds == 0


def test_scatter_spills(ctx):
    """A key that carries 45 % of the rows overflows its lanes: those rows are claimed by k_spill's general path."""
    n = (1 << 20) + 1021
    fold = _fold(ctx, n=n)
    try:
        st = _run(fold, _batches(nb=2, n=n, hot_key=77))
    finally:
        fold.close()
    assert st.combined_folds == 2 and st.scatter_spill_rows > 0


@pytest.mark.parametrize("split", [True, False])
def test_late_rows(ctx, monkeypatch, split):
    """Activations with late rows: split off (the rest on the segment fold), or the whole activation on the sort path."""
    monkeypatch.setenv("BW_LATE_SPLIT", "1" if split else "0")
    fold = _fold(ctx, wait=S)
    try:
        st = _run(fold, _batches(late_every=997))
    finally:
        fold.close()
    if split:
        assert st.split_batches == 2
    else:
        assert st.slow_batches == 2


def test_restore(ctx):
    batches = _batches(nb=4)
    fold = _fold(ctx)
    try:
        for keys, ts, vals in batches[:2]:
            fold.ingest(keys, vals, ts)
            fold.advance()
        snap = fold.snapshot()
    finally:
        fold.close()
    fold = _fold(ctx)
    try:
        fold.restore(snap)
        seen = set(snap["key"].tolist())
        assert seen
        _check(fold, seen)
        for keys, ts, vals in batches[2:]:
            fold.ingest(keys, vals, ts)
            seen.update(keys.tolist())
            _check(fold, seen)
    finally:
        fold.close()


@pytest.mark.parametrize("world", [2, 4])
def test_loopback_world(world):
    """World > 1 on one device: every rank's table is claimed by the merge-at-owner pass (k_segfold MODE 2)."""
    from bytewax_b200 import _native as N, gpu
    from oracle import pyoracle as po

    ctxs = gpu.Context.loopback_world(world)
    per_rank = [_batches(nb=3, n=1 << 15, seed=11 + r) for r in range(world)]
    got, errors, folds = [None] * world, [None] * world, [None] * world

    def rank_main(r):
        try:
            # (wait: the ranks' slices of an activation overlap in event time; none of their rows is late)
            fold = folds[r] = gpu.WindowFold(ctxs[r], "sum", 2 * S, None, A, 5 * S, val_dtype="i64", capacity_hint=1 << 17,
                                             max_batch_rows=1 << 15, max_emit_rows=1 << 22, max_late_rows=1 << 18,
                                             exchange=N.XCHG_P2P)
            for keys, ts, vals in per_rank[r]:
                fold.ingest(keys, vals, ts)
            fold.advance()
            got[r] = (fold.check_key_column(), int(fold.stats().combined_folds))
        except BaseException as ex:  # noqa: BLE001 - reported by the main thread
            errors[r] = ex

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for f in folds:
        if f is not None:
            f.close()
    for c in ctxs:
        c.close()
    for ex in errors:
        if ex is not None:
            raise ex
    owner = [po.dest_rank(k, world) for k in set(np.concatenate([k for b in per_rank for k, _, _ in b]).tolist())]
    for r in range(world):
        (bad, used), combined = got[r]
        assert bad == 0 and combined > 0
        assert used == owner.count(r)
