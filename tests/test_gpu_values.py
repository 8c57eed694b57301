"""The window fold at the limits of its value types, against oracle/exact.py.  Needs an H100: -m gpu.

The emission sequence (which (key, window) rows, in which activation, in which order) comes from the C oracle, fed the
values as 64-bit integer bits or binary64 (the order never depends on the values); every accumulator is compared with
the exact one: integers and min / max bit for bit, float sums and means against the error bound of binary64 summation
in any order (which a single rounding to binary32 anywhere exceeds).  Every test runs in both fold modes."""

import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import coracle, exact  # noqa: E402  (checker only)

S = 1_000_000
A = 1_640_995_200_000_000
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
FLOAT = ("f32", "f64")


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


def _inorder(seed, nb=3, n=50_000, n_keys=2000, span_us=8 * S):
    """Keys and non-decreasing timestamps of `nb` activations: windows stay open across activations."""
    rnd = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        ts = (A - 3 * S + b * span_us + (np.arange(n) * span_us) // n).astype(np.int64)
        out.append((rnd.integers(0, n_keys, n).astype(np.uint64), ts))
    return rnd, out


def _oracle_vals(vals, dtype):
    return vals.astype(np.float64) if dtype in FLOAT else vals.view(np.int64)


def _run(ctx, red, dtype, length, offset, batches, wait=0, n_keys=2000):
    """Every activation through the fold (advance after each) and the C oracle; rows and oracle columns."""
    from bytewax_b200 import gpu

    n = max(len(k) for k, _, _ in batches)
    fold = gpu.WindowFold(ctx, red, length * S, offset * S if offset else None, A, wait * S, val_dtype=dtype,
                          capacity_hint=max(4096, n_keys), max_batch_rows=n, max_emit_rows=1 << 20, max_late_rows=1 << 18)
    orc = coracle.COracle("count", length * S, offset * S if offset else None, A, wait * S, False, is_float=dtype in FLOAT)
    ems = []
    for keys, ts, vals in batches:
        fold.ingest(keys, vals, ts)
        orc.on_batch(keys, ts, _oracle_vals(vals, dtype))
        ems.append(fold.advance())
    ems.append(fold.eof())
    orc.on_eof()
    st = fold.stats()
    fold.close()
    ck, cw, _, _, cact = orc.closed()
    late = orc.late()
    orc.close()
    cat = lambda f: np.concatenate([getattr(e, f) for e in ems])  # noqa: E731
    for b, e in enumerate(ems):  # each activation's rows, in the oracle's order
        sel = cact == b
        assert np.array_equal(e.closed_key, ck[sel]) and np.array_equal(e.closed_window_id, cw[sel]), b
    got = {f: cat(f) for f in ("closed_key", "closed_window_id", "closed_acc", "closed_count", "late_key", "late_window_id",
                               "late_val", "late_ts_us")}
    assert len(got["closed_key"]) > 1000  # not vacuous
    return got, late, st


def _check_acc(got, want, red, dtype):
    keys, wids, acc = got["closed_key"].tolist(), got["closed_window_id"].tolist(), got["closed_acc"]
    assert sorted(zip(keys, wids)) == sorted(want)
    exp = [want[kw] for kw in zip(keys, wids)]
    if red == "mean" or (red == "sum" and dtype in FLOAT):
        fs = np.array([e.fsum for e in exp])
        bound = np.array([e.bound() for e in exp])
        err = np.abs(acc - fs)
        bad = ~(err <= bound)
        assert not bad.any(), (int(bad.sum()), acc[bad][:4], fs[bad][:4], bound[bad][:4])
        assert np.isfinite(acc[np.isfinite(fs)]).all()  # no binary32 overflow on the way
        if red == "mean":
            assert got["closed_count"].tolist() == [e.n for e in exp]
    elif dtype in FLOAT:  # min / max: bit for bit
        assert np.array_equal(acc.view(np.uint64), np.array(exp, np.float64).view(np.uint64))
    else:
        assert acc.dtype == (np.int64 if dtype == "i64" and red != "count" else np.uint64)
        assert acc.tolist() == exp


def _check_stats(st, fold_mode, nb):
    assert st.slow_batches == 0
    assert st.combined_folds == (nb if fold_mode == "stream" else 0)


def _fold_and_check(ctx, fold_mode, red, dtype, length, offset, batches, n_keys=2000):
    got, _, st = _run(ctx, red, dtype, length, offset, batches, n_keys=n_keys)
    _check_acc(got, exact.fold(red, length * S, offset * S if offset else None, A, 0, batches, dtype), red, dtype)
    _check_stats(st, fold_mode, len(batches))
    return got


WINDOWS = [(10, None), (10, 5)]  # tumbling; sliding (two panes per window: combined at close time)


@pytest.mark.parametrize("length,offset", WINDOWS)
def test_i64_sum_wraps_and_carries(ctx, fold_mode, length, offset):
    """Values whose low words carry on nearly every add and whose window sums leave the i64 range."""
    edge = np.array([2**62, -(2**62), I64_MAX, -I64_MAX, 0xFFFFFFFF, 2**32, -1], np.int64)
    rnd, kt = _inorder(11)
    batches = [(k, t, rnd.choice(edge, len(k))) for k, t in kt]
    _fold_and_check(ctx, fold_mode, "sum", "i64", length, offset, batches)
    # not vacuous: many windows' unbounded sums leave the i64 range (the exact ones above are those wrapped)
    unbounded = exact.fold("sum", length * S, offset * S if offset else None, A, 0,
                           [(k, t, v.astype(np.float64)) for k, t, v in batches], "f64")
    assert sum(1 for e in unbounded.values() if abs(e.fsum) >= 2.0**63) > 100


@pytest.mark.parametrize("red", ["sum", "min", "max"])
@pytest.mark.parametrize("length,offset,n_keys", [(10, None, 2000), (10, 5, 2000), (10, None, 100_000)])
def test_u64_whole_range(ctx, fold_mode, red, length, offset, n_keys):
    """u64 values over the whole range, half of them >= 2^63: a signed op picks a different min / max."""
    rnd, kt = _inorder(12, n_keys=n_keys)
    edge = np.array([0, 1, 2**63 - 1, 2**63, 2**64 - 1], np.uint64)
    batches = []
    for k, t in kt:
        v = rnd.integers(0, 2**64 - 1, len(k), dtype=np.uint64, endpoint=True)
        pick = rnd.random(len(k)) < 0.1
        v[pick] = rnd.choice(edge, int(pick.sum()))
        batches.append((k, t, v))
    _fold_and_check(ctx, fold_mode, red, "u64", length, offset, batches, n_keys=n_keys)


@pytest.mark.parametrize("red", ["min", "max"])
@pytest.mark.parametrize("length,offset", WINDOWS)
def test_i64_identity_values(ctx, fold_mode, red, length, offset):
    """Windows whose only value is the accumulator's identity (INT64_MAX for min, INT64_MIN for max), and keys whose
    first pane of every window holds only the identity while the second holds ordinary values: such rows are emitted
    with that value, never dropped or mistaken for an empty pane."""
    ident = I64_MAX if red == "min" else I64_MIN
    rnd, kt = _inorder(13)
    batches = []
    for k, t in kt:
        v = rnd.integers(-1000, 1000, len(k))
        cls = k % np.uint64(4)
        v[cls == 0] = ident
        first_pane = ((t - A) // (5 * S)) % 2 == 0
        v[(cls == 1) & first_pane] = ident
        batches.append((k, t, v))
    got = _fold_and_check(ctx, fold_mode, red, "i64", length, offset, batches)
    assert (got["closed_acc"] == ident).sum() > 100


def _float_edges(dtype):
    fi = np.finfo(np.float32 if dtype == "f32" else np.float64)
    tiny = float(fi.smallest_subnormal)
    return np.array([math.inf, -math.inf, float(fi.max), -float(fi.max), tiny, -tiny, 3 * tiny, float(fi.smallest_normal),
                     -float(fi.smallest_normal), -1.5, 2.5])


@pytest.mark.parametrize("dtype", FLOAT)
@pytest.mark.parametrize("red", ["min", "max"])
@pytest.mark.parametrize("length,offset", WINDOWS)
def test_float_min_max_bits(ctx, fold_mode, red, dtype, length, offset):
    """Negatives, infinities, the largest finite values and subnormals through the ordered encoding: bit for bit."""
    rnd, kt = _inorder(14)
    edge = _float_edges(dtype)
    batches = []
    for k, t in kt:
        v = rnd.normal(0, 1e3, len(k))
        pick = rnd.random(len(k)) < 0.08
        v[pick] = rnd.choice(edge, int(pick.sum()))
        v[k % np.uint64(5) == 0] = -np.abs(v[k % np.uint64(5) == 0])  # keys with negative values only
        batches.append((k, t, v.astype(np.float32 if dtype == "f32" else np.float64)))
    _fold_and_check(ctx, fold_mode, red, dtype, length, offset, batches)


def _zero_batches(red, seed=15):
    """Keys whose windows mix -0.0 and +0.0 (with negatives for max, positives for min: a zero is the result)."""
    rnd, kt = _inorder(seed)
    batches = []
    for k, t in kt:
        v = np.where(rnd.random(len(k)) < 0.5, -0.0, 0.0)
        other = rnd.random(len(k)) < 0.3
        v[other] = rnd.uniform(1, 100, int(other.sum())) * (-1 if red == "max" else 1)
        only_neg = k % np.uint64(7) == 0  # ... and keys with -0.0 only, +0.0 only
        only_pos = k % np.uint64(7) == 1
        v[only_neg], v[only_pos] = -0.0, 0.0
        batches.append((k, t, v))
    return batches


def _device_zero_rule(red, batches, length, offset):
    """The device's documented signed-zero rule (DESIGN.md section 10): min and max order -0.0 below +0.0, so a max
    that compares equal to zero is +0.0 when the window holds a +0.0 and a min is -0.0 when it holds a -0.0, whatever
    the arrival order.  (The reference keeps the first zero that arrived.)"""
    want = exact.fold(red, length * S, offset * S if offset else None, A, 0, batches, "f64")
    sign = -0.0 if red == "min" else 0.0
    marks = [(k, t, (np.signbit(v) == np.signbit(sign)) & (v == 0)) for k, t, v in batches]
    has = exact.fold("max", length * S, offset * S if offset else None, A, 0, [(k, t, m.astype(np.float64)) for k, t, m in marks], "f64")
    return {kw: (math.copysign(0.0, -1.0 if red == "min" else 1.0) if x == 0 and has[kw] == 1.0 else x) for kw, x in want.items()}


@pytest.mark.parametrize("red", ["min", "max"])
@pytest.mark.parametrize("length,offset", WINDOWS)
def test_signed_zeros(ctx, fold_mode, red, length, offset):
    batches = _zero_batches(red)
    got, _, st = _run(ctx, red, "f64", length, offset, batches)
    keys, wids = got["closed_key"].tolist(), got["closed_window_id"].tolist()
    ref = exact.fold(red, length * S, offset * S if offset else None, A, 0, batches, "f64")
    assert got["closed_acc"].tolist() == [ref[kw] for kw in zip(keys, wids)]  # == the reference's value (as numbers)
    dev = _device_zero_rule(red, batches, length, offset)
    want_bits = np.array([dev[kw] for kw in zip(keys, wids)], np.float64).view(np.uint64)
    assert np.array_equal(got["closed_acc"].view(np.uint64), want_bits)
    neg = np.signbit(got["closed_acc"]) & (got["closed_acc"] == 0)
    assert 0 < int(neg.sum()) < len(neg)  # both zeros come out
    _check_stats(st, fold_mode, len(batches))


def _sum_values(rnd, k, dtype):
    n = len(k)
    cls = (k % np.uint64(3)).astype(np.int64)
    v = rnd.normal(0, 1e3, n)
    if dtype == "f64":
        # class 1: 1e8, x, -1e8 (cancellation); class 2: magnitudes from 1e-3 to 1e6, random signs
        pat = np.resize(np.array([1e8, 0.0, -1e8]), n)
        v = np.where(cls == 1, np.where(pat == 0.0, rnd.normal(0, 1, n), pat), v)
        v = np.where(cls == 2, 10.0 ** rnd.uniform(-3, 6, n) * rnd.choice([-1.0, 1.0], n), v)
        return v
    # class 1: near the top of the f32 range, mostly positive: window sums exceed it
    v = np.where(cls == 1, rnd.uniform(2.5e38, 3.4e38, n) * np.where(rnd.random(n) < 0.9, 1.0, -1.0), v)
    return v.astype(np.float32)


@pytest.mark.parametrize("dtype", FLOAT)
@pytest.mark.parametrize("red", ["sum", "mean"])
@pytest.mark.parametrize("length,offset", WINDOWS)
def test_float_sum_mean_error_bound(ctx, fold_mode, red, dtype, length, offset):
    """Mixed signs and magnitudes: |got - fsum| <= n u sum|x| (binary64 in any order), no inf where the exact sum is
    finite (f32 inputs whose sums pass 3.4e38), exact counts for mean."""
    rnd, kt = _inorder(16)
    batches = [(k, t, _sum_values(rnd, k, dtype)) for k, t in kt]
    got = _fold_and_check(ctx, fold_mode, red, dtype, length, offset, batches)
    if dtype == "f32":
        assert (np.abs(got["closed_acc"]) > float(np.finfo(np.float32).max)).sum() > 10  # not vacuous


@pytest.mark.parametrize("red,dtype", [("max", "u64"), ("sum", "i64"), ("min", "f32")])
def test_late_rows_keep_their_value_bits(ctx, fold_mode, red, dtype):
    """A few rows per activation arrive 40 s behind their key's previous row (late with wait 0); their values are edge
    values, returned in the late stream bit for bit.  The closed windows are those of the other rows."""
    rnd, kt = _inorder(17)
    batches, clean = [], []
    for k, t in kt:
        n = len(k)
        if dtype == "u64":
            v = rnd.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
            edge = np.array([2**64 - 1, 2**63, 2**63 + 1, 0], np.uint64)
        elif dtype == "i64":
            v = rnd.integers(-1000, 1000, n)
            edge = np.array([I64_MIN, I64_MAX, -1, 2**32], np.int64)
        else:
            v = rnd.normal(0, 1e3, n).astype(np.float32)
            edge = np.array([float(np.finfo(np.float32).max), -math.inf, float(np.finfo(np.float32).smallest_subnormal), 0.1],
                            np.float32)
        k, t = k.copy(), t.copy()
        at = np.sort(rnd.choice(np.arange(1, n), 40, replace=False))
        k[at] = k[at - 1]
        t[at] = t[at - 1] - 40 * S
        v[at] = rnd.choice(edge, len(at))
        batches.append((k, t, v))
        keep = np.ones(n, bool)
        keep[at] = False
        clean.append((k[keep], t[keep], v[keep]))
    got, (lk, lw, lv, lts, _), st = _run(ctx, red, dtype, 10, None, batches)
    _check_acc(got, exact.fold(red, 10 * S, None, A, 0, clean, dtype), red, dtype)
    assert len(lk) >= 100
    assert got["late_key"].tolist() == lk.tolist() and got["late_window_id"].tolist() == lw.tolist()
    assert got["late_ts_us"].tolist() == lts.tolist()
    want_bits = lv.view(np.uint64)
    assert np.array_equal(got["late_val"].view(np.uint64), want_bits)
    if fold_mode == "stream":
        assert st.split_batches == len(batches) and st.slow_batches == 0


def _loopback_values(rnd, kind, n):
    if kind == "u64":
        return rnd.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    if kind == "mixed":
        return rnd.normal(0, 1e3, n) * np.where(rnd.random(n) < 0.5, 1.0, 1e6)
    v = np.where(rnd.random(n) < 0.5, -0.0, 0.0)
    v[rnd.random(n) < 0.2] = -3.0 if kind == "zeros_max" else 3.0
    return v


@pytest.mark.parametrize("red,dtype,kind", [("max", "u64", "u64"), ("sum", "f64", "mixed"), ("max", "f64", "zeros_max"),
                                            ("min", "f64", "zeros_min")])
def test_loopback_world_values(fold_mode, red, dtype, kind):
    """World 2 on one device: the partials `k_segfold<1>` stores at the source and `<2>` merges at the owner carry the
    values exactly (u64 max, mixed-sign f64 sums, signed zeros -- the same bits as one rank)."""
    from tests.test_gpu_loopback import make_batches, oracle_rows, run_world

    world = 2
    rnd = np.random.default_rng(18)
    batches = [[(k, t, _loopback_values(rnd, kind, len(k))) for k, t, _ in per_rank] for per_rank in make_batches(world, "inorder")]
    got = run_world(world, red, 10, None, 0, batches, val_dtype=dtype)
    flat = [(np.concatenate([p[r][0] for r in range(world)]), np.concatenate([p[r][1] for r in range(world)]),
             np.concatenate([p[r][2] for r in range(world)])) for p in batches]
    if kind.startswith("zeros"):
        want = _device_zero_rule(red, flat, 10, None)
    else:
        want = exact.fold(red, 10 * S, None, A, 0, flat, dtype)
    zeros = [[(k, t, np.zeros(len(k), np.int64)) for k, t, _ in per_rank] for per_rank in batches]
    total = 0
    for d in range(world):
        (ck, cw, _, _, _), _ = oracle_rows(world, d, "count", 10, None, 0, zeros)
        g = got[d]
        assert g["ck"].tolist() == ck.tolist() and g["cw"].tolist() == cw.tolist(), d
        sub = {kw: want[kw] for kw in zip(ck.tolist(), cw.tolist())}
        _check_acc(dict(closed_key=g["ck"], closed_window_id=g["cw"], closed_acc=g["ca"]), sub, red, dtype)
        if fold_mode == "stream":
            assert g["stream"] == len(batches)
        total += len(ck)
    assert total == len(want)
