"""The `*_final` folds (`ts_source == BW_TS_NONE`) at the limits of their values, keys, paths and worlds.  -m gpu.

A final fold keeps one accumulator per key and emits nothing before EOF; EOF emits every key once, as window 0, in
ascending key-string order.  Every accumulator is compared with `oracle/exact.py` as Python objects: integers and
min / max bit for bit, float sums and means against the error bound of binary64 summation in any order (which a single
rounding to binary32 anywhere exceeds).  Every test runs in both fold modes and asserts through `bw_stats` the path it
took: the segment fold (`combined_folds`), the direct kernel, or lanes spilled by a hot key (`scatter_spill_rows`)."""

import ctypes as C
import math
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import exact, pyoracle as po  # noqa: E402  (checker only)

S = 1_000_000
A = 1_640_995_200_000_000
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
U64_MAX = 2**64 - 1
FLOAT = ("f32", "f64")
REDS = ("count", "sum", "min", "max", "mean")
DTYPES = ("i64", "u64", "f32", "f64")
NV = (1 << 20) + 1023  # rows per activation: the last 2048-row tile is partial, and not a multiple of 4
NK = 20_000


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module", params=["stream", "direct"], autouse=True)
def fold_mode(request):
    """Streaming path (bucket scatter + shared-memory segment fold) and the direct hash-table kernel alone."""
    old = os.environ.get("BW_STREAM")
    os.environ["BW_STREAM"] = "1" if request.param == "stream" else "0"
    yield request.param
    if old is None:
        os.environ.pop("BW_STREAM", None)
    else:
        os.environ["BW_STREAM"] = old


def _make(ctx, red, dtype, cap, rows, emit=1 << 20):
    from bytewax_b200 import gpu

    return gpu.WindowFold(ctx, red, val_dtype=dtype, final=True, capacity_hint=cap, max_batch_rows=rows, max_emit_rows=emit,
                          max_late_rows=1 << 10)


def _nothing(em):
    return em.closed_key.size == 0 and em.late_key.size == 0


def _run(ctx, red, dtype, batches, cap=NK, emit=1 << 20):
    """Every activation through one final fold; nothing may come out before EOF, also not from a notify phase."""
    fold = _make(ctx, red, dtype, cap, max(len(k) for k, _ in batches), emit)
    try:
        for i, (keys, vals) in enumerate(batches):
            fold.ingest(keys, vals)
            assert _nothing(fold.advance(system_now_us=A + i * S if i % 2 else 0)), i
        em = fold.eof()
        return em, fold.stats()
    finally:
        fold.close()


def _check(em, want, red, dtype, zero_rule=None):
    """EOF rows == the exact accumulators of `want` (key -> accumulator), in ascending key-string order, window 0."""
    keys = em.closed_key.tolist()
    assert keys == sorted(want, key=str)
    assert em.closed_window_id.tolist() == [0] * len(keys)
    exp = [want[k] for k in keys]
    got = em.closed_acc.tolist()
    if red == "mean" or (red == "sum" and dtype in FLOAT):
        bad = [(k, g, e.fsum, e.bound()) for k, g, e in zip(keys, got, exp) if not abs(g - e.fsum) <= e.bound()]
        assert not bad, (len(bad), bad[:4])
        assert all(math.isfinite(g) for g, e in zip(got, exp) if math.isfinite(e.fsum))  # no binary32 overflow
        if red == "mean":
            assert em.closed_count.tolist() == [e.n for e in exp]
    elif dtype in FLOAT and red != "count":  # min / max: bit for bit
        assert got == exp  # == the reference's values, as numbers
        if zero_rule is not None:
            exp = [zero_rule(k, e) for k, e in zip(keys, exp)]
        assert em.closed_acc.view(np.uint64).tolist() == np.array(exp, np.float64).view(np.uint64).tolist()
    else:
        assert type(got[0]) is int and got == exp


def _check_stats(st, fold_mode, nb):
    assert st.slow_batches == 0
    assert st.combined_folds == (nb if fold_mode == "stream" else 0)


# ---------------------------------------------------------------------------- values


def _float_edges(dtype):
    fi = np.finfo(np.float32 if dtype == "f32" else np.float64)
    tiny = float(fi.smallest_subnormal)
    return np.array([math.inf, -math.inf, float(fi.max), -float(fi.max), tiny, -tiny, 3 * tiny, float(fi.smallest_normal),
                     -float(fi.smallest_normal), -0.0, 0.0, -1.5, 2.5])


def _values(rnd, k, red, dtype):
    n = len(k)
    if dtype == "i64":  # low words that carry, sums that leave the range both ways, the extremes themselves
        v = rnd.integers(I64_MIN, I64_MAX, n, endpoint=True)
        edge = np.array([I64_MIN, I64_MAX, 2**62, -(2**62), -I64_MAX, 0xFFFFFFFF, 2**32, -1, 0, 1], np.int64)
        pick = rnd.random(n) < 0.3
        v[pick] = rnd.choice(edge, int(pick.sum()))
        return v
    if dtype == "u64":  # the whole range, half of it >= 2^63 (a signed op picks a different min / max)
        v = rnd.integers(0, U64_MAX, n, dtype=np.uint64, endpoint=True)
        pick = rnd.random(n) < 0.2
        v[pick] = rnd.choice(np.array([0, 1, 2**63 - 1, 2**63, U64_MAX], np.uint64), int(pick.sum()))
        return v
    np_t = np.float32 if dtype == "f32" else np.float64
    cls = (k % np.uint64(7)).astype(np.int64)
    if red in ("sum", "mean"):  # a wide dynamic range: one rounding to binary32 anywhere is far outside the bound
        v = rnd.normal(0, 1e3, n)
        if dtype == "f64":
            pat = np.resize(np.array([1e8, 0.0, -1e8]), n)
            v = np.where(cls == 1, np.where(pat == 0.0, rnd.normal(0, 1, n), pat), v)
            v = np.where(cls == 2, 10.0 ** rnd.uniform(-3, 6, n) * rnd.choice([-1.0, 1.0], n), v)
            v = np.where(cls == 3, 1.0 + rnd.integers(1, 2**20, n) * 2.0**-40, v)  # bits below binary32's mantissa
        else:  # near the top of the binary32 range, mostly positive: sums pass it
            v = np.where(cls == 1, rnd.uniform(2.5e38, 3.4e38, n) * np.where(rnd.random(n) < 0.9, 1.0, -1.0), v)
        v[cls == 4] = -0.0  # a sum of -0.0 alone is +0.0 on the device (identity +0.0); -0.0 == +0.0
        return v.astype(np_t)
    v = rnd.normal(0, 1e3, n)
    pick = rnd.random(n) < 0.1
    v[pick] = rnd.choice(_float_edges(dtype), int(pick.sum()))
    zeros = np.where(rnd.random(n) < 0.5, -0.0, 0.0)  # signed zeros where a zero is the result
    v = np.where(cls == 0, zeros, v)  # zeros only
    v = np.where((cls == 1) & (rnd.random(n) < 0.5), zeros, np.where(cls == 1, np.abs(v) + 1, v))  # zeros and positives
    v = np.where((cls == 2) & (rnd.random(n) < 0.5), zeros, np.where(cls == 2, -np.abs(v) - 1, v))  # zeros and negatives
    v[(cls == 3) & (k % np.uint64(2) == 0)] = -0.0  # -0.0 only, and +0.0 only
    v[(cls == 3) & (k % np.uint64(2) == 1)] = 0.0
    return v.astype(np_t)


def _value_batches(red, dtype, nb=3):
    rnd = np.random.default_rng(100 + 10 * DTYPES.index(dtype) + REDS.index(red))
    out = []
    for _ in range(nb):
        k = rnd.integers(0, NK, NV).astype(np.uint64)
        out.append((k, _values(rnd, k, red, dtype)))
    return out


_WANT = {}  # (red, dtype) -> exact accumulators, shared by both fold modes


def _zero_rule(red, batches):
    """The device's documented signed-zero rule (DESIGN.md section 10): min and max order -0.0 below +0.0, so a max that
    compares equal to zero is +0.0 when the key holds a +0.0 and a min is -0.0 when it holds a -0.0, whatever the
    arrival order.  (The reference keeps the first zero that arrived.)"""
    held = set()
    for k, v in batches:
        v = v.astype(np.float64)
        held.update(k[(v == 0) & (np.signbit(v) == (red == "min"))].tolist())
    return lambda k, x: (math.copysign(0.0, -1.0 if red == "min" else 1.0) if k in held else x) if x == 0 else x


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("red", REDS)
def test_values(ctx, fold_mode, red, dtype):
    """Every reduction over every value type: 3 activations of 2^20 + 1023 rows over 20 000 keys, accumulators carried
    across activations.  No (reduction, value type) pair is refused by the spec."""
    batches = _value_batches(red, dtype)
    if (red, dtype) not in _WANT:
        _WANT[red, dtype] = exact.final(red, batches, dtype)
    want = _WANT[red, dtype]
    em, st = _run(ctx, red, dtype, batches)
    zr = _zero_rule(red, batches) if dtype in FLOAT and red in ("min", "max") else None
    _check(em, want, red, dtype, zr)
    _check_stats(st, fold_mode, len(batches))
    acc = em.closed_acc
    if zr is not None:  # both zeros come out, and the device's sign differs from the reference's somewhere
        zero = acc == 0
        assert 0 < int((zero & np.signbit(acc)).sum()) < int(zero.sum())
        ref_neg = [math.copysign(1.0, want[k]) < 0 for k in em.closed_key[zero].tolist()]
        assert ref_neg != np.signbit(acc[zero]).tolist()
    if red == "sum" and dtype in FLOAT:
        keys = em.closed_key.tolist()
        only_neg0 = [i for i, k in enumerate(keys) if k % 7 == 4]
        # a key whose only value is -0.0 sums to +0.0 here (identity +0.0) where the host keeps -0.0: they compare equal
        assert only_neg0 and all(acc[i] == 0 and not np.signbit(acc[i]) for i in only_neg0)
        if dtype == "f32":  # not vacuous: sums past the binary32 range, finite here
            assert sum(abs(want[k].fsum) > float(np.finfo(np.float32).max) for k in keys) > 100
        else:  # not vacuous: rounding the exact sum to binary32 is outside the bound
            assert sum(abs(float(np.float32(e.fsum)) - e.fsum) > e.bound() for e in want.values()) > 1000
    if red == "sum" and dtype == "i64":  # not vacuous: sums that wrapped
        assert sum(1 for e in want.values() if abs(e) > 2**62) > 1000


# ---------------------------------------------------------------------------- keys and emission order


def _digit_keys():
    ks = list(range(10))
    for k in range(1, 20):
        ks += [10**k - 1, 10**k]
    ks += [10**19 + d for d in range(10)]  # 20 digits: they share their first 19
    ks += [2**63 - 1, 2**63, U64_MAX]  # U64_MAX: the table's empty-slot alias
    return ks


def test_keys_and_emission_order(ctx, fold_mode):
    """Every digit-count class, the 20-digit keys that differ in the last digit only, the signed / unsigned boundary,
    the empty-slot alias and 10^5 random full-range keys, in shuffled order: EOF is ascending key-string order."""
    rnd = np.random.default_rng(7)
    keys = np.unique(np.concatenate([np.array(_digit_keys(), np.uint64),
                                     rnd.integers(0, U64_MAX, 100_000, dtype=np.uint64, endpoint=True)]))
    rows = rnd.permutation(np.repeat(keys, 3))
    batches = []
    for part in np.array_split(rows, 3):
        batches.append((part, rnd.integers(-1000, 1000, len(part))))
    for red in ("count", "sum"):
        em, st = _run(ctx, red, "i64", batches, cap=len(keys))
        _check(em, exact.final(red, batches, "i64"), red, "i64")
        _check_stats(st, fold_mode, len(batches))
        head = [k for k in em.closed_key.tolist() if k >= 10**19 and k < 10**19 + 10]
        assert head == [10**19 + d for d in range(10)]


# ---------------------------------------------------------------------------- scale, skew, staging


def test_scale_1e6_keys(ctx, fold_mode):
    """About 10^6 keys over 4 activations of 2^21 rows (count and i64 sum), checked with numpy: segments filled as C1's."""
    rnd = np.random.default_rng(8)
    n, nk = 1 << 21, 1_000_000
    batches = [(rnd.integers(0, nk, n).astype(np.uint64), rnd.integers(-2**40, 2**40, n)) for _ in range(4)]
    k = np.concatenate([b[0] for b in batches])
    v = np.concatenate([b[1] for b in batches])
    uk, inv = np.unique(k, return_inverse=True)
    assert len(uk) > 990_000
    order = np.argsort(uk.astype(str), kind="stable")
    sums = np.zeros(len(uk), np.int64)
    np.add.at(sums, inv, v)
    for red, want in (("count", np.bincount(inv)), ("sum", sums)):
        em, st = _run(ctx, red, "i64", batches, cap=nk)
        assert em.closed_key.tolist() == uk[order].tolist()
        assert em.closed_window_id.tolist() == [0] * len(uk)
        assert em.closed_acc.tolist() == want[order].tolist()
        _check_stats(st, fold_mode, len(batches))


def _skewed(shape, seed, nb=2, n=(1 << 20) + 1021, n_keys=100_000):
    rnd = np.random.default_rng(seed)
    out = []
    for _ in range(nb):
        if shape == "zipf":
            keys = rnd.zipf(1.1, n)
            keys = np.where(keys <= n_keys, keys - 1, rnd.integers(0, n_keys, n))
        else:
            keys = rnd.integers(0, n_keys, n)
            keys[rnd.random(n) < 0.45] = 77  # one key carries 45 % of the rows
        out.append(keys.astype(np.uint64))
    return rnd, out


_SKEW_WANT = {}


@pytest.mark.parametrize("red,dtype", [("count", "i64"), ("sum", "i64"), ("sum", "f64")])
@pytest.mark.parametrize("shape", ["hot", "zipf"])
def test_skewed_keys_spill(ctx, fold_mode, shape, red, dtype):
    """A hot key (45 % of every activation) and Zipf(1.1) over 10^5 keys: the streaming path spills the lanes that
    overflow, and no row is lost or counted twice."""
    rnd, keys = _skewed(shape, 21)
    batches = [(k, rnd.normal(0, 1e3, len(k)) if dtype == "f64" else rnd.integers(-1000, 1000, len(k))) for k in keys]
    if (shape, red, dtype) not in _SKEW_WANT:
        _SKEW_WANT[shape, red, dtype] = exact.final(red, batches, dtype)
    em, st = _run(ctx, red, dtype, batches, cap=100_000)
    _check(em, _SKEW_WANT[shape, red, dtype], red, dtype)
    _check_stats(st, fold_mode, len(batches))
    if fold_mode == "stream":
        assert st.scatter_spill_rows > 0


# pairwise points of test_gpu_stream_paths' (BW_SC_STG, BW_SC_EVERY, BW_SC_STAGES, BW_SEG_SHIFT) matrix
STAGING = [(0, 1, 2, 10), (4, None, 3, 11), (8, 1000, 4, 12), (16, 1, 3, 12), (16, None, 2, 11), (6, 1000, 2, 10)]


@pytest.mark.parametrize("stg,every,stages,seg", STAGING)
def test_staging_matrix_count(ctx, fold_mode, monkeypatch, stg, every, stages, seg):
    """A count final fold (`k_scatter<2, 0, 0>`, the one staged final instantiation) under staging depths, write-out
    cadences, TMA stage counts and segment sizes, one hot bucket included."""
    if fold_mode == "direct":
        pytest.skip("the scatter settings shape the streaming path only")
    for name, v in (("BW_SC_STG", stg), ("BW_SC_EVERY", every), ("BW_SC_STAGES", stages), ("BW_SEG_SHIFT", seg)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))
    rnd = np.random.default_rng(stg * 100 + stages * 10 + seg)
    batches = []
    for _ in range(2):
        k = rnd.integers(0, 100_000, NV).astype(np.uint64)
        k[rnd.random(NV) < 0.1] = 12345
        batches.append((k, None))
    em, st = _run(ctx, "count", "u64", batches, cap=100_000)
    uk, cnt = np.unique(np.concatenate([b[0] for b in batches]), return_counts=True)
    _check(em, dict(zip(uk.tolist(), cnt.tolist())), "count", "u64")
    _check_stats(st, fold_mode, len(batches))


# ---------------------------------------------------------------------------- device columns


@pytest.mark.parametrize("red,dtype", [("count", "u64"), ("sum", "i64"), ("sum", "f32"), ("max", "f64")])
def test_device_columns(ctx, fold_mode, red, dtype):
    """Columns already on the device (`bw_ingest_device`): 16-byte aligned ones take the streaming path, the same rows
    one element past an aligned address take the direct kernel (`combined_folds == 0`); both give the same EOF rows."""
    rnd = np.random.default_rng(9)
    n = NV
    np_t = {"u64": np.uint64, "i64": np.int64, "f32": np.float32, "f64": np.float64}[dtype]
    batches = []
    for _ in range(3):
        k = rnd.integers(0, NK, n).astype(np.uint64)
        v = (rnd.normal(0, 1e3, n) * 10.0 ** rnd.integers(-3, 4, n) if dtype in FLOAT else rnd.integers(0, 2**40, n)).astype(np_t)
        batches.append((k, v))
    want = exact.final(red, batches, dtype)
    vb = np.dtype(np_t).itemsize
    for shift in (0, 1):
        fold = _make(ctx, red, dtype, NK, n)
        bufs = []
        try:
            for k, v in batches:
                dk, dv = ctx.dev_alloc((n + 1) * 8), ctx.dev_alloc((n + 1) * vb)
                bufs += [dk, dv]
                ctx.h2d(dk + shift * 8, k)
                ctx.h2d(dv + shift * vb, v)
                fold.ingest_device(dk + shift * 8, dv + shift * vb, None, n)
                assert _nothing(fold.advance())
            em = fold.eof()
            st = fold.stats()
        finally:
            fold.close()
            for p in bufs:
                ctx.dev_free(p)
        _check(em, want, red, dtype)
        assert st.slow_batches == 0
        assert st.combined_folds == (len(batches) if fold_mode == "stream" and shift == 0 else 0), shift


# ---------------------------------------------------------------------------- worlds


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


def _run_world(world, red, dtype, batches, snap=None, cap=NK, rows=1 << 16):
    """`batches[b][r]` is source rank r's slice of activation b; every rank restores `snap` first when given.  Returns
    per rank its EOF rows and stats; nothing may come out of any rank before EOF."""
    from bytewax_b200 import gpu

    ctxs = gpu.Context.loopback_world(world)
    folds = [None] * world

    def rank_main(r):
        f = folds[r] = _make(ctxs[r], red, dtype, cap, rows)
        if snap is not None:
            f.restore(snap)
        for b, per_rank in enumerate(batches):
            f.ingest(*per_rank[r])
            assert _nothing(f.advance()), (r, b)
        return f.eof(), f.stats()

    try:
        return _in_threads(world, rank_main)
    finally:
        for f in folds:  # every rank is done with its peers' memory: only now free anything
            if f is not None:
                f.close()
        for c in ctxs:
            c.close()


def _dest(keys, world):
    return {k: po.dest_rank(k, world) for k in set(keys)}


def _world_values(rnd, dtype, n):
    if dtype == "u64":
        return rnd.integers(0, U64_MAX, n, dtype=np.uint64, endpoint=True)
    if dtype == "f64":
        return rnd.normal(0, 1e3, n) * np.where(rnd.random(n) < 0.5, 1.0, 1e6)
    return rnd.integers(I64_MIN, I64_MAX, n, endpoint=True)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("red,dtype", [("count", "i64"), ("sum", "i64"), ("sum", "f64"), ("max", "u64")])
def test_loopback_world(fold_mode, world, red, dtype):
    """Worlds of 2 and 4 ranks on one device: each rank's EOF rows are exactly the keys the route gives it, in
    key-string order, with exact accumulators.  Streaming: combine at the source and merge at the owner every
    activation; BW_STREAM=0: the row exchange and the direct kernel."""
    rnd = np.random.default_rng(10 + world)
    n, nb = 1 << 16, 3
    batches = [[(rnd.integers(0, NK, n).astype(np.uint64) * np.uint64(7919), _world_values(rnd, dtype, n))
                for _ in range(world)] for _ in range(nb)]
    flat = [kv for per_rank in batches for kv in per_rank]
    want = exact.final(red, flat, dtype)
    dest = _dest(want, world)
    got = _run_world(world, red, dtype, batches)
    for d, (em, st) in enumerate(got):
        mine = {k: e for k, e in want.items() if dest[k] == d}
        assert len(mine) > NK // world // 2
        _check(em, mine, red, dtype)
        _check_stats(st, fold_mode, nb)


# ---------------------------------------------------------------------------- limits and states


def test_emit_limit_at_eof(ctx, fold_mode):
    """EOF emits every key at once: exactly `max_emit_rows` keys fit, one more is BW_ERR_CAPACITY."""
    from bytewax_b200 import _native as N

    m = 5000
    keys = np.arange(m + 1, dtype=np.uint64) * np.uint64(1_000_003)
    em, _ = _run(ctx, "count", "u64", [(keys[:m], None)], cap=8192, emit=m)
    _check(em, {k: 1 for k in keys[:m].tolist()}, "count", "u64")
    fold = _make(ctx, "count", "u64", 8192, m + 1, emit=m)
    try:
        fold.ingest(keys, None)
        assert _nothing(fold.advance())
        with pytest.raises(N.BwError) as e:
            fold.eof()
        assert e.value.status == 3
    finally:
        fold.close()


def test_more_keys_than_the_table_raises(ctx, fold_mode):
    from bytewax_b200 import _native as N

    fold = _make(ctx, "sum", "i64", 2048, 1 << 14)
    try:
        assert fold.stats().table_capacity == 4096
        keys = np.arange(1 << 14, dtype=np.uint64) * np.uint64(7919)
        with pytest.raises(N.BwError) as e:
            fold.ingest(keys, np.ones(1 << 14, np.int64))
            fold.advance()
        assert e.value.status == 3
    finally:
        fold.close()


def test_empty_activations_and_eof_states(ctx, fold_mode):
    """An empty activation emits nothing and changes nothing; an EOF with no rows at all emits nothing; a second EOF and
    an ingest after EOF are BW_ERR_STATE."""
    from bytewax_b200 import _native as N

    empty = (np.zeros(0, np.uint64), np.zeros(0, np.int64))
    fold = _make(ctx, "sum", "i64", 1024, 1024)
    try:
        fold.ingest(*empty)
        assert _nothing(fold.advance())
        em = fold.eof()
        assert _nothing(em)
        with pytest.raises(N.BwError) as e:
            fold.eof()
        assert e.value.status == 5
        with pytest.raises(N.BwError) as e:
            fold.ingest(np.array([1], np.uint64), np.array([1], np.int64))
        assert e.value.status == 5
    finally:
        fold.close()
    batches = [(np.array([5, 10, 9], np.uint64), np.array([I64_MAX, -1, 2], np.int64)), empty,
               (np.array([10, 5], np.uint64), np.array([1, 1], np.int64)), empty]
    em, st = _run(ctx, "sum", "i64", batches, cap=1024)
    assert em.closed_key.tolist() == [10, 5, 9]
    assert em.closed_acc.tolist() == [0, I64_MIN, 2]
    assert st.slow_batches == 0


def test_ts_none_needs_wait_forever(ctx):
    """`BW_TS_NONE` with a finite wait is BW_ERR_SPEC; with `BW_WAIT_FOREVER` the same spec creates a fold."""
    from bytewax_b200 import _native as N

    def create(wait):
        s = N.BwFoldSpec()
        s.struct_size = C.sizeof(N.BwFoldSpec)
        s.reduction, s.val_dtype, s.ts_source = N.RED["count"], N.VAL["u64"], N.TS_NONE
        s.length_us = s.offset_us = S
        s.align_to_us, s.wait_us = A, wait
        s.exchange, s.ring_slots = N.XCHG_P2P, 3
        s.capacity_hint = s.max_batch_rows = s.max_emit_rows = s.max_late_rows = 1024
        h = C.c_void_p()
        st = ctx.lib.bw_fold_create(ctx.h, C.byref(s), C.byref(h))
        if h:
            ctx.lib.bw_fold_destroy(h)
        return st

    assert create(0) == 4 and create(5 * S) == 4
    assert create(N.BW_WAIT_FOREVER) == 0


# ---------------------------------------------------------------------------- snapshot


@pytest.mark.parametrize("red,dtype", [("count", "i64"), ("sum", "i64"), ("max", "u64"), ("sum", "f64")])
def test_snapshot_restore(ctx, fold_mode, red, dtype):
    """A snapshot between activations, restored into a fresh final fold of a smaller and of a larger table and into a
    loopback world of 2: the resumed EOF rows equal the uninterrupted fold's (float sums: the same exact bound)."""
    rnd = np.random.default_rng(12)
    n, nb, cut = 1 << 16, 4, 2
    batches = [(rnd.integers(0, 5000, n).astype(np.uint64) * np.uint64(104_729), _world_values(rnd, dtype, n)) for _ in range(nb)]
    want = exact.final(red, batches, dtype)
    whole, _ = _run(ctx, red, dtype, batches, cap=8192)
    _check(whole, want, red, dtype)
    a = _make(ctx, red, dtype, 8192, n)
    try:
        for k, v in batches[:cut]:
            a.ingest(k, v)
            assert _nothing(a.advance())
        snap = a.snapshot()
    finally:
        a.close()
    assert len(snap["key"]) == 5000 and set(snap["pane_id"].tolist()) <= {0}
    for cap in (5000, 1 << 16):
        b = _make(ctx, red, dtype, cap, n)
        try:
            b.restore(snap)
            for k, v in batches[cut:]:
                b.ingest(k, v)
                assert _nothing(b.advance())
            em = b.eof()
        finally:
            b.close()
        _check(em, want, red, dtype)
        if not (red == "sum" and dtype == "f64"):
            assert em.closed_acc.tolist() == whole.closed_acc.tolist()
    halves = [[(k[: n // 2], v[: n // 2]), (k[n // 2:], v[n // 2:])] for k, v in batches[cut:]]
    got = _run_world(2, red, dtype, halves, snap=snap)
    dest = _dest(want, 2)
    for d, (em, st) in enumerate(got):
        _check(em, {k: e for k, e in want.items() if dest[k] == d}, red, dtype)
        assert st.slow_batches == 0
