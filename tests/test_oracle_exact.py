"""oracle/exact.py (the unbounded-precision accumulators behind tests/test_gpu_values.py) against the C oracle and the
reference's stored rows, on inputs where both are exact: nothing wraps, nothing is late."""

import json
import math
import os

import numpy as np
import pytest

from oracle import coracle, exact

S = 1_000_000
A = 1_640_995_200_000_000


def _inorder_batches(seed, is_float, nb=4, n=3000, n_keys=300, span_us=7 * S):
    rnd = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        ts = (A - 13 * S + b * span_us + (np.arange(n) * span_us) // n).astype(np.int64)
        keys = rnd.integers(0, n_keys, n).astype(np.uint64)
        vals = rnd.normal(0, 1e3, n) if is_float else rnd.integers(-10**6, 10**6, n)
        out.append((keys, ts, vals))
    return out


def _check_float_sum(got, want: exact.FloatSum, where):
    assert abs(got - want.fsum) <= want.bound(), where


@pytest.mark.parametrize("is_float", [False, True])
@pytest.mark.parametrize("red", ["count", "sum", "min", "max", "mean"])
@pytest.mark.parametrize("length,offset", [(5, None), (10, 4)])
def test_exact_equals_c_oracle_inorder(red, is_float, length, offset):
    batches = _inorder_batches(hash((red, is_float, length)) & 0xFFFF, is_float)
    orc = coracle.COracle(red, length * S, offset * S if offset else None, A, 0, False, is_float=is_float)
    for keys, ts, vals in batches:
        orc.on_batch(keys, ts, vals)
    orc.on_eof()
    ck, cw, ca, cc, _ = orc.closed()
    want = exact.fold(red, length * S, offset * S if offset else None, A, 0, batches, "f64" if is_float else "i64")
    assert sorted(zip(ck.tolist(), cw.tolist())) == sorted(want)  # the same (key, window) set
    for k, w, a, c in zip(ck.tolist(), cw.tolist(), ca.tolist(), cc.tolist()):
        e = want[(k, w)]
        if red == "mean":
            assert c == e.n
            _check_float_sum(a, e, (k, w))
        elif red == "sum" and is_float:
            _check_float_sum(a, e, (k, w))
        else:
            assert a == e, (k, w)


def test_exact_equals_clean_golden_cases(golden_dir):
    """Every stored case without late rows: the reference's own accumulators (Python ints / floats summed left to right)."""
    with open(os.path.join(golden_dir, "window_fold_cases.json")) as f:
        cases = json.load(f)
    checked = 0
    for name, case in cases.items():
        if any(t == "L" for act in case["acts"] for _k, _w, t, _p in act):
            continue
        s = case["spec"]
        is_float = any(isinstance(v, float) for b in case["batches"] for v in b[2])
        want = exact.fold(s["reduction"], s["length_us"], s["offset_us"], s["align_us"], s["wait_us"],
                          [(k, t, v) for k, t, v in case["batches"]], "f64" if is_float else "i64")
        rows = [(k, w, p) for act in case["acts"] for k, w, t, p in act if t == "E"]
        assert sorted((k, w) for k, w, _ in rows) == sorted(want), name
        for k, w, p in rows:
            e = want[(k, w)]
            if isinstance(e, exact.FloatSum):
                if s["reduction"] == "mean":
                    assert p[1] == e.n
                    p = p[0]
                _check_float_sum(p, e, (name, k, w))
            else:
                assert p == e and type(p) is type(e), (name, k, w)
        checked += 1
    assert checked >= 8


def test_exact_rules_at_the_limits():
    def one(red, dtype, vals, ts=None):
        ts = ts or [A] * len(vals)
        return exact.fold(red, 10 * S, None, A, 0, [([7] * len(vals), ts, vals)], dtype)[(7, 0)]

    # integer sums wrap mod 2^64 and are read back with the dtype's signedness
    assert one("sum", "i64", [2**63 - 1, 1]) == -(2**63)
    assert one("sum", "i64", [-(2**63), -1]) == 2**63 - 1
    assert one("sum", "u64", [2**64 - 1, 2]) == 1
    assert one("sum", "u64", [2**63, 2**63, 5]) == 5
    # unsigned order is not signed order
    assert one("max", "u64", [2**63, 5]) == 2**63 and one("min", "u64", [2**63, 5]) == 5
    # the first of equal values stays: the sign of a zero result is the first zero's
    for red in ("min", "max"):
        assert math.copysign(1.0, one(red, "f64", [-0.0, 0.0])) == -1.0
        assert math.copysign(1.0, one(red, "f64", [0.0, -0.0])) == 1.0
    assert one("max", "f64", [-math.inf, -1e308]) == -1e308 and one("min", "f64", [math.inf, 5e-324]) == 5e-324
    # an f32 value counts as the binary64 value it widens to
    f = np.array([0.1, 3e38], np.float32)
    assert one("max", "f32", f) == float(f[1]) and one("min", "f32", f) == float(np.float64(f[0]))
    # f32 values whose sum leaves the f32 range: the sum is the binary64 one
    s = one("sum", "f32", np.array([3e38, 3e38, -1.0], np.float32))
    assert math.isfinite(s.fsum) and s.fsum == math.fsum([float(np.float32(3e38))] * 2 + [-1.0]) and s.n == 3
    # the error bound admits f64 summation in any order but not one rounding to f32
    xs = np.random.default_rng(3).normal(0, 1e3, 60).tolist() + [1e8, 1.0 + 2**-30, -1e8] * 20
    e = one("sum", "f64", xs)
    assert abs(sum(xs) - e.fsum) <= e.bound() and abs(sum(reversed(xs)) - e.fsum) <= e.bound()
    assert abs(math.fsum(float(np.float32(x)) for x in xs) - e.fsum) > e.bound()
    # a value out of the dtype's range and a row that may be late are refused
    with pytest.raises(ValueError):
        one("sum", "i64", [2**63])
    with pytest.raises(ValueError):
        one("count", "i64", [1, 1], ts=[A + 5 * S, A + 4 * S])


@pytest.mark.parametrize("dtype", ["i64", "u64", "f32", "f64"])
@pytest.mark.parametrize("red", ["count", "sum", "min", "max", "mean"])
def test_final_is_fold_in_window_zero(red, dtype):
    """`exact.final` (the *_final folds' accumulators, grouped by a numpy sort) equals `exact.fold` with every row at the
    align: the same value and type per key, the same zero sign for min / max, in any number of batches."""
    rnd = np.random.default_rng(7)
    batches = []
    for n in (500, 1, 700):
        keys = rnd.choice(np.array([0, 1, 9, 10, 2**63, 2**64 - 1], np.uint64), n)
        if dtype == "i64":
            vals = rnd.choice(np.array([-(2**63), 2**63 - 1, -1, 0, 5], np.int64), n)
        elif dtype == "u64":
            vals = rnd.choice(np.array([0, 1, 2**63, 2**64 - 1], np.uint64), n)
        else:
            edge = [-0.0, 0.0, -1.5, 2.5, 5e-324] + ([math.inf, -math.inf] if red in ("min", "max") else [])
            vals = rnd.choice(np.array(edge), n)
            vals = vals.astype(np.float32 if dtype == "f32" else np.float64)
        batches.append((keys, vals))
    want = exact.fold(red, 10 * S, None, A, None, [(k, np.full(len(k), A), v) for k, v in batches], dtype)
    got = exact.final(red, batches, dtype)
    assert {w for _k, w in want} == {0}
    assert list(got) == sorted(got) and set(got) == {k for k, _w in want}
    for k, e in got.items():
        assert e == want[(k, 0)] and type(e) is type(want[(k, 0)]), k
        if isinstance(e, float):
            assert math.copysign(1.0, e) == math.copysign(1.0, want[(k, 0)]), k
