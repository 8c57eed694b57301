"""K7: session-window folds on the device (`bw_session_*`) against the reference's own session windower.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/session_cases.json (made by the reference's
`_WindowLogic` + `_SessionWindowerLogic`, tools/gen_session_golden.py) including the bits of every f64 accumulator and
the merged ids, the SHA-256 digests of its seeded streams, and `tests/session_oracle.run_sessions` on larger streams."""

import json
import math
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import session_oracle as so

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = so.S, so.A
SENTINEL = 2**64 - 1


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _fold(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    return gpu.SessionFold(ctx, spec["reduction"], spec["gap_us"], None if wait == so.WAIT_FOREVER else wait,
                           val_dtype=spec.get("val_dtype", "i64"), **kw)


def _key_text_ordered(keys):
    text = [str(k) for k in keys]
    return text == sorted(text)


def _rows(out, batch):
    """Device rows of one call as the reference's row list: per key its late rows, then E / M per closed session.  The
    device's own order is checked, not restored: each of the late and closed columns must already come in ascending
    key-string order (src/operators.rs:758-767), late rows in arrival order and sessions in id order within a key; the two
    columns are then interleaved key by key in that order.  Late rows get their value back from the input row they name."""
    lk, lr, la = out.late_key.tolist(), out.late_row.tolist(), out.late_activation.tolist()
    ck, cw = out.closed_key.tolist(), out.closed_window_id.tolist()
    assert _key_text_ordered(lk) and _key_text_ordered(ck), "device rows not in ascending key-string order"
    assert all(lk[i] != lk[i + 1] or lr[i] < lr[i + 1] for i in range(len(lk) - 1)), "late rows not in arrival order"
    assert all(ck[i] != ck[i + 1] or cw[i] < cw[i + 1] for i in range(len(ck) - 1)), "sessions not in id order"
    late = []
    for k, act, r in zip(lk, la, lr):
        assert batch is not None and act == batch[0]
        late.append((k, [k, -1, "L", batch[1][r]]))
    closed = []
    for i, (k, w, a, o, c) in enumerate(zip(ck, cw, out.closed_acc.tolist(), out.closed_open_us.tolist(), out.closed_close_us.tolist())):
        closed.append((k, [k, w, "E", a]))
        closed.append((k, [k, w, "M", [o, c, out.merged(i)]]))
    rows, i, j = [], 0, 0
    while i < len(late) or j < len(closed):  # merge of two key-ordered lists; a key's late rows come first
        if j == len(closed) or (i < len(late) and str(late[i][0]) <= str(closed[j][0])):
            rows.append(late[i][1])
            i += 1
        else:
            rows.append(closed[j][1])
            j += 1
    return rows


def run_device(ctx, spec, steps, **kw):
    """Drive a SessionFold through golden-format steps; rows per step, then EOF."""
    f = _fold(ctx, spec, **kw)
    acts, n_act = [], 0
    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                _, now, keys, ts, vals = step
                dt = np.float64 if spec.get("val_dtype") == "f64" else np.int64
                f.apply(np.array(keys, dtype=np.uint64), None if spec["reduction"] == "count" else np.array(vals, dtype=dt),
                        np.array(ts, dtype=np.int64), epoch=i + 1, system_now_us=now)
                acts.append(_rows(f.advance(), (n_act, vals)))
                n_act += 1
            else:
                acts.append(_rows(f.advance(system_now_us=step[1]), None))
        acts.append(_rows(f.eof(), None))
    finally:
        f.close()
    return acts


def _same(a, b):
    """Exact equality where floats compare by bits (any NaN equals any NaN: payloads are not part of the contract)."""
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))
    if isinstance(a, list) and isinstance(b, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return type(a) is type(b) and a == b


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "session_cases.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case(ctx, golden, name):
    case = golden["cases"][name]
    got = run_device(ctx, case["spec"], case["steps"])
    assert _same(got, case["acts"]), (got, case["acts"])


@pytest.mark.parametrize("seed", list(so.SEEDED))
def test_seeded_digests(ctx, golden, seed):
    spec, steps = so.seeded_steps(seed, moving=seed % 3 != 0)
    got = run_device(ctx, spec, steps, max_sessions_per_key=64)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]


def _big_stream(seed, n_act, rows, n_keys, hot_rows=0, fval=False):
    rnd = np.random.default_rng(seed)
    steps, base, now = [], A, A + 100 * S
    for b in range(n_act):
        keys = rnd.integers(0, n_keys, rows).astype(np.uint64)
        keys[rnd.random(rows) < 0.001] = SENTINEL
        if hot_rows:
            keys[:hot_rows] = 7
        ts = base + rnd.integers(-6 * S, 6 * S, rows) - np.where(rnd.random(rows) < 0.05, rnd.integers(5 * S, 40 * S, rows), 0)
        vals = rnd.choice(np.array(so.F64_VALUES), rows) if fval else rnd.integers(-1000, 1000, rows)
        now += int(rnd.integers(0, 2 * S))
        steps.append(["batch", now, keys.tolist(), ts.tolist(), vals.tolist()])
        if b % 2:
            steps.append(["notify", now + 3 * S])
        base += 3 * S
    return steps


@pytest.mark.parametrize("seed,red,dtype", [(1, "count", "i64"), (2, "sum", "f64"), (3, "max", "i64"), (4, "min", "f64")])
def test_random_streams_match_oracle(ctx, seed, red, dtype):
    spec = dict(reduction=red, val_dtype=dtype, gap_us=1 * S, wait_us=2 * S)
    steps = _big_stream(seed, 6, 40_000, 3000, fval=dtype == "f64")
    want = so.run_sessions(spec, steps)
    got = run_device(ctx, spec, steps, capacity_hint=1 << 13, max_batch_rows=1 << 16, max_sessions_per_key=64)
    merges = sum(len(r[3][2]) for a in want for r in a if r[2] == "M")
    lates = sum(r[2] == "L" for a in want for r in a)
    assert merges > 1000 and lates > 1000
    for i, (g, w) in enumerate(zip(got, want)):
        assert _same(g, w), f"step {i}"
    assert len(got) == len(want)


def test_hot_key_serial(ctx):
    """One key with 10^5 items per activation next to 20 000 light keys."""
    spec = dict(reduction="sum", val_dtype="i64", gap_us=S // 2, wait_us=S)
    steps = _big_stream(5, 3, 150_000, 20_000, hot_rows=100_000)
    want = so.run_sessions(spec, steps)
    got = run_device(ctx, spec, steps, capacity_hint=1 << 15, max_batch_rows=1 << 18, max_sessions_per_key=64)
    assert _same(got, want)


# ---------------------------------------------------------------------------
# capacity and spec edges
# ---------------------------------------------------------------------------


def _expect_capacity(fn, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == 3 and what in str(ei.value), str(ei.value)


def test_key_table_exactly_full(ctx):
    from bytewax_b200 import gpu

    f = gpu.SessionFold(ctx, "count", S, 0, capacity_hint=16)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, SENTINEL], dtype=np.uint64)
        ts = np.full(keys.size, A, dtype=np.int64)
        f.apply(keys, None, ts, system_now_us=1)
        f.apply(keys, None, ts + 10 * S, system_now_us=1)  # every key closes its first session
        out = f.advance()
        assert out.closed_key.size == 1025 and (out.closed_acc == 1).all()
        _expect_capacity(lambda: f.apply(np.array([2000, 2001], np.uint64), None, np.array([A, A], np.int64)), "key table full")
        with pytest.raises(N.BwError) as ei:
            f.advance()
        assert ei.value.status == 5
    finally:
        f.close()


def test_sessions_per_key_exactly_full(ctx):
    from bytewax_b200 import gpu

    f = gpu.SessionFold(ctx, "count", 5 * S, None, max_sessions_per_key=4)
    try:
        f.apply(np.array([3, 3, 3, 3], np.uint64), None, np.array([A, A + 20 * S, A + 40 * S, A + 60 * S], np.int64))
        # session 0 grows to A + 15 s and absorbs session 1: three live sessions, one merged id held
        f.apply(np.array([3, 3, 3], np.uint64), None, np.array([A + 5 * S, A + 10 * S, A + 15 * S], np.int64))
        f.apply(np.array([3], np.uint64), None, np.array([A + 80 * S], np.int64))  # four live again
        assert f.advance().closed_key.size == 0
        _expect_capacity(lambda: f.apply(np.array([3], np.uint64), None, np.array([A + 100 * S], np.int64)), "max_sessions_per_key")
    finally:
        f.close()
    f = gpu.SessionFold(ctx, "count", 5 * S, None, max_sessions_per_key=4)
    try:
        f.apply(np.array([3, 3, 3, 3], np.uint64), None, np.array([A, A + 20 * S, A + 40 * S, A + 60 * S], np.int64))
        f.apply(np.array([3, 3, 3], np.uint64), None, np.array([A + 5 * S, A + 10 * S, A + 15 * S], np.int64))
        out = f.eof()
        assert out.closed_window_id.tolist() == [0, 2, 3] and out.merged(0) == [1] and out.closed_acc.tolist() == [5, 1, 1]
    finally:
        f.close()


def test_emit_and_late_buffers_exactly_full(ctx):
    from bytewax_b200 import gpu

    f = gpu.SessionFold(ctx, "sum", S, 0, max_emit_rows=10, max_late_rows=5)
    try:
        keys = np.arange(10, dtype=np.uint64)
        f.apply(keys, np.arange(10), np.full(10, A, np.int64))
        f.apply(keys, np.arange(10), np.full(10, A + 10 * S, np.int64))  # closes 10 sessions
        f.apply(keys[:5], np.zeros(5), np.full(5, A, np.int64))  # 5 lates
        out = f.advance()
        assert out.closed_key.size == 10 and out.late_key.size == 5
        assert out.closed_acc.tolist() == list(range(10)) and out.late_row.tolist() == list(range(5))
        _expect_capacity(lambda: f.apply(keys[:6], np.zeros(6), np.full(6, A, np.int64)), "max_late_rows")
    finally:
        f.close()
    f = gpu.SessionFold(ctx, "count", S, 0, max_emit_rows=10)
    try:
        keys = np.arange(11, dtype=np.uint64)
        f.apply(keys, None, np.full(11, A, np.int64))
        _expect_capacity(lambda: f.apply(keys, None, np.full(11, A + 10 * S, np.int64)), "max_emit_rows")
    finally:
        f.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(val_dtype="u64"), dict(val_dtype="f32"), dict(gap_us=-1), dict(wait_us=-1), dict(max_sessions_per_key=0),
               dict(max_sessions_per_key=65), dict(reduction="mean"), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as ei:
            gpu.SessionFold(ctx, **kw)
        assert ei.value.status == 4, kw
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as ei:
            gpu.SessionFold(ctxs[0])
        assert ei.value.status == 4 and "one GPU" in str(ei.value)
    finally:
        for c in ctxs:
            c.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle():
        f = gpu.SessionFold(ctx, "sum", S, 0, val_dtype="f64", capacity_hint=1 << 18, max_sessions_per_key=32)
        rnd = random.Random(1)
        keys = np.array([rnd.randrange(5000) for _ in range(20000)], np.uint64)
        f.apply(keys, np.ones(keys.size), A + np.arange(keys.size, dtype=np.int64) * 1000)
        f.advance(system_now_us=A + 100 * S)
        f.eof()
        f.close()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    cycle()
    before = free()
    for _ in range(3):
        cycle()
    assert before - free() < (32 << 20)
