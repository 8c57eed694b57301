"""K11: `max_window` / `min_window` with ``by=`` on the device (`bw_argwin_*`) against the reference's own rows.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/arg_window_cases.json (made by
the reference's `_WindowLogic` + windower + `_FoldWindowLogic`, tools/gen_arg_window_golden.py), the SHA-256 digests of
its seeded streams, and `tests/arg_window_oracle.run_arg_window` on larger streams -- including the handles each call
releases."""

import json
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import arg_window_oracle as aw

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = aw.S, aw.A
SENTINEL = 2**64 - 1
UTC_MAX = 253_402_300_799_999_999


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _is_f64(steps) -> bool:
    return any(isinstance(aw.dec(b), float) for s in steps if s[0] == "batch" for b in s[4])


def _arg(ctx, spec, f64, **kw):
    from bytewax_b200 import gpu

    wait = None if spec["wait_us"] == aw.WAIT_FOREVER else spec["wait_us"]
    kw.setdefault("max_windows_per_key", 64)
    if "gap_us" in spec:
        return gpu.ArgWindow(ctx, spec["extreme"], "f64" if f64 else "i64", gap_us=spec["gap_us"], wait_us=wait, **kw)
    return gpu.ArgWindow(ctx, spec["extreme"], "f64" if f64 else "i64", spec["length_us"], spec["offset_us"], spec["align_us"],
                         wait_us=wait, **kw)


def _groups(keys, what):
    """Runs of equal keys, checked to come in ascending key-string order (src/operators.rs:758-767), each key once."""
    runs = []
    for i, k in enumerate(keys):
        if runs and runs[-1][0] == k:
            runs[-1][1].append(i)
        else:
            runs.append((k, [i]))
    text = [str(k) for k, _ in runs]
    assert text == sorted(text) and len(set(text)) == len(text), f"{what} rows not in ascending key-string order"
    return dict(runs)


def _rows(out, batch, session):
    """Device rows of one call as the reference's row list: per key its late rows (arrival order), then an `E` and an
    `M` row per closed window in the device's order."""
    lk, lw, lr, la = out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist(), out.late_activation.tolist()
    ck, cw, ch = out.closed_key.tolist(), out.closed_window_id.tolist(), out.closed_handle.tolist()
    co, cc = out.closed_open_us.tolist(), out.closed_close_us.tolist()
    gl, gc = _groups(lk, "late"), _groups(ck, "closed")
    rows = []
    for k in sorted(set(gl) | set(gc), key=str):
        for i in gl.get(k, []):
            assert batch is not None and la[i] == batch["act"]
            rows.append([k, lw[i], "L", batch["handles"][lr[i]]])
        for i in gc.get(k, []):
            rows.append([k, cw[i], "E", ch[i]])
            rows.append([k, cw[i], "M", [co[i], cc[i], out.merged(i)] if session else [co[i], cc[i]]])
            if not session:
                assert out.merged(i) == []
    return rows


def _cols(step, f64):
    _, _now, keys, ts, bys, handles = step
    return (np.array(keys, dtype=np.uint64), np.array(handles, dtype=np.uint64),
            np.array([aw.dec(b) for b in bys], dtype=np.float64 if f64 else np.int64), np.array(ts, dtype=np.int64))


def run_device(ctx, spec, steps, device_cols=False, f64=None, **kw):
    """Drive an ArgWindow through golden-format steps: (rows, sorted released handles) per step, then EOF."""
    f64 = _is_f64(steps) if f64 is None else f64
    a = _arg(ctx, spec, f64, **kw)
    session = "gap_us" in spec
    acts, released, n_act = [], [], 0

    def take(out, batch):
        acts.append(_rows(out, batch, session))
        released.append(sorted(out.released.tolist()))

    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                cols = _cols(step, f64)
                if device_cols:
                    d = [torch.from_numpy(c.view(np.int64) if c.dtype == np.uint64 else c).cuda() for c in cols]
                    a.apply_device(*(t.data_ptr() for t in d), len(step[2]), epoch=i + 1, system_now_us=step[1])
                    out = a.advance()  # (waits for the call: the columns stay alive until then)
                    del d
                else:
                    a.apply(*cols, epoch=i + 1, system_now_us=step[1])
                    out = a.advance()
                take(out, dict(act=n_act, handles=step[5]))
                n_act += 1
            else:
                take(a.advance(system_now_us=step[1]), None)
        take(a.eof(), None)
    finally:
        a.close()
    return acts, released


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "arg_window_cases.json")


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case(ctx, golden, name):
    case = golden["cases"][name]
    got, released = run_device(ctx, case["spec"], case["steps"])
    assert got == case["acts"]
    assert released == aw.run_arg_window(case["spec"], case["steps"])[1]


@pytest.mark.parametrize("seed", list(aw.SEEDED))
def test_seeded_digests(ctx, golden, seed):
    spec, steps = aw.seeded_steps(seed, moving=seed % 3 != 1)
    got, released = run_device(ctx, spec, steps, f64=(seed // 12) % 2 == 1)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]
    assert released == aw.run_arg_window(spec, steps)[1]


def test_apply_device_matches_apply(ctx):
    for seed in (0, 13, 26, 38):
        spec, steps = aw.seeded_steps(seed)
        f64 = (seed // 12) % 2 == 1
        assert run_device(ctx, spec, steps, device_cols=True, f64=f64) == run_device(ctx, spec, steps, f64=f64)


def _spec(windower, extreme, wait=S):
    if windower == "session":
        return dict(extreme=extreme, gap_us=2 * S, wait_us=wait)
    length, offset = (4 * S, 4 * S) if windower == "tumbling" else (6 * S, 2 * S)
    return dict(extreme=extreme, length_us=length, offset_us=offset, align_us=A + 123, wait_us=wait)


@pytest.mark.parametrize("windower", aw.WINDOWERS)
@pytest.mark.parametrize("extreme", ["max", "min"])
@pytest.mark.parametrize("f64", [False, True])
def test_random_streams_match_oracle(ctx, windower, extreme, f64):
    """1000 keys, late rows, a moving clock with notify phases, every handle released once."""
    seed = 100 + aw.WINDOWERS.index(windower) * 4 + ("max", "min").index(extreme) * 2 + int(f64)
    _, steps = aw.seeded_steps(seed, n_steps=24, n_keys=1000, f64=f64, max_items=2000)
    spec = _spec(windower, extreme)
    got, rel = run_device(ctx, spec, steps, f64=f64, capacity_hint=1 << 11, max_batch_rows=1 << 14)
    want, want_rel = aw.run_arg_window(spec, steps)
    assert got == want
    assert rel == want_rel
    assert any(r[2] == "L" for act in got for r in act) and any(s[0] == "notify" for s in steps)
    flat = [h for r in rel for h in r]
    assert len(flat) == len(set(flat)) == sum(len(s[5]) for s in steps if s[0] == "batch")


def _first_best(by, extreme):
    return int(np.argmax(by) if extreme == "max" else np.argmin(by))  # (numpy's: the FIRST best index)


@pytest.mark.parametrize("extreme", ["max", "min"])
@pytest.mark.parametrize("windower", ["tumbling", "sliding"])
def test_hot_key_one_million_values(ctx, windower, extreme):
    """10^6 values of one key in one tumbling window, or in six sliding windows (60 s / 10 s), with many ties."""
    n = 1_000_000
    rng = np.random.default_rng(5)
    by = rng.integers(-1000, 1000, n, dtype=np.int64)
    if windower == "tumbling":
        spec = dict(extreme=extreme, length_us=3600 * S, offset_us=3600 * S, align_us=A, wait_us=None)
        ts = A + np.arange(n, dtype=np.int64)
    else:
        spec = dict(extreme=extreme, length_us=60 * S, offset_us=10 * S, align_us=A, wait_us=None)
        ts = A + 55 * S + (np.arange(n, dtype=np.int64) % (5 * S))  # every value in windows 0..5
    a = _arg(ctx, dict(spec, wait_us=aw.WAIT_FOREVER), False, capacity_hint=16, max_batch_rows=n)
    try:
        a.apply(np.full(n, 7, np.uint64), np.arange(n, dtype=np.uint64), by, ts)
        out = a.advance()
        want = _first_best(by, extreme)
        # every handle released once: the losers in the call that received them, the pick at its last window's close
        assert out.closed_key.size == 0 and out.released.size == n - 1 and want not in set(out.released.tolist())
        out = a.eof()
        nwin = 1 if windower == "tumbling" else 6
        assert out.closed_handle.tolist() == [want] * nwin
        assert out.closed_window_id.tolist() == list(range(nwin))
        assert out.released.tolist() == [want]
    finally:
        a.close()


def test_hot_key_one_long_session(ctx):
    """10^5 values of one key, 1 us apart with gap 2 s: one session."""
    n = 100_000
    rng = np.random.default_rng(6)
    by = rng.normal(size=n)
    a = _arg(ctx, dict(extreme="min", gap_us=2 * S, wait_us=aw.WAIT_FOREVER), True, capacity_hint=16, max_batch_rows=n)
    try:
        perm = rng.permutation(n)  # out of order: every item extends or lands in the one session
        a.apply(np.full(n, 9, np.uint64), np.arange(n, dtype=np.uint64), by, A + perm.astype(np.int64))
        out = a.eof()
        assert out.closed_window_id.tolist() == [0] and out.closed_handle.tolist() == [int(np.argmin(by))]
        assert [out.closed_open_us[0], out.closed_close_us[0]] == [A, A + n - 1]
    finally:
        a.close()


# ---------------------------------------------------------------------------
# capacity and spec edges
# ---------------------------------------------------------------------------


def _expect(fn, status, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == status and what in str(ei.value), str(ei.value)


def _refused(a):
    with pytest.raises(N.BwError) as ei:
        a.advance()
    assert ei.value.status == 5


def _mk(ctx, session=False, **kw):
    from bytewax_b200 import gpu

    args = dict(extreme="max", by_dtype="i64", wait_us=0)
    args.update(dict(gap_us=S) if session else dict(length_us=10 * S, align_us=A))
    args.update(kw)
    return gpu.ArgWindow(ctx, **args)


@pytest.mark.parametrize("session", [False, True])
def test_key_table_exactly_full(ctx, session):
    a = _mk(ctx, session, capacity_hint=16)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, SENTINEL], dtype=np.uint64)
        ts = np.full(keys.size, A, np.int64)
        a.apply(keys, np.arange(keys.size), np.zeros(keys.size), ts)
        assert a.advance().closed_key.size == 0
        a.apply(keys, np.arange(keys.size) + 5000, np.ones(keys.size), ts + 20 * S)  # every key closes its first window
        out = a.advance()
        assert out.closed_key.size == 1025 and sorted(out.closed_handle.tolist()) == list(range(1025))
        assert sorted(out.released.tolist()) == list(range(1025))
        _expect(lambda: a.apply(np.array([2000, 2001], np.uint64), np.array([1, 2]), np.zeros(2), np.array([A, A], np.int64) + 20 * S),
                3, "key table full")
        _refused(a)
    finally:
        a.close()


@pytest.mark.parametrize("session", [False, True])
def test_windows_per_key_exactly_full(ctx, session):
    for extra, ok in ((0, True), (1, False)):
        a = _mk(ctx, session, wait_us=None, max_windows_per_key=4, **({"gap_us": 0} if session else {}))
        try:
            n = 4 + extra
            call = lambda: a.apply(np.full(n, 3, np.uint64), np.arange(n), np.arange(n), A + np.arange(n, dtype=np.int64) * 10 * S)  # noqa: E731
            if ok:
                call()
                out = a.eof()
                assert out.closed_window_id.tolist() == [0, 1, 2, 3] and sorted(out.released.tolist()) == [0, 1, 2, 3]
            else:
                _expect(call, 3, "max_windows_per_key")
                _refused(a)
        finally:
            a.close()


def test_merged_ids_exactly_full(ctx):
    """M = 3: a survivor holds 3 merged ids; a fourth merge into it fails."""
    for extra, ok in ((0, True), (1, False)):
        a = _mk(ctx, True, gap_us=10 * S, wait_us=None, max_windows_per_key=3)
        try:
            def one(x, y, h):  # a new session at x, then y extends it to within gap of session 0: one merge per call
                a.apply(np.array([5, 5], np.uint64), np.array([h, h + 1]), np.array([h, h + 1]), np.array([x, y], np.int64))

            one(A, A, 0)
            for c in range(3):
                one(A + (20 + 20 * c) * S, A + (10 + 20 * c) * S, 2 * c + 2)
            assert a.advance().closed_key.size == 0
            if ok:
                out = a.eof()
                assert out.closed_window_id.tolist() == [0] and out.merged(0) == [1, 2, 3] and out.closed_handle.tolist() == [7]
                assert sorted(out.released.tolist()) == [7]
            else:
                _expect(lambda: one(A + 80 * S, A + 70 * S, 10), 3, "merged ids")
                _refused(a)
        finally:
            a.close()


@pytest.mark.parametrize("session", [False, True])
def test_emit_and_late_buffers_exactly_full(ctx, session):
    a = _mk(ctx, session, max_emit_rows=10, max_late_rows=5)
    try:
        a.apply(np.arange(10, dtype=np.uint64), np.arange(10), np.arange(10), np.full(10, A + 5 * S, np.int64))
        a.apply(np.arange(5, dtype=np.uint64), np.arange(5) + 10, np.arange(5), np.full(5, A - 20 * S, np.int64))  # 5 lates
        out = a.advance()
        assert out.late_key.size == 5 and out.late_row.tolist() == list(range(5))
        assert sorted(out.released.tolist()) == list(range(10, 15))
        out = a.eof()
        assert out.closed_key.size == 10
    finally:
        a.close()
    a = _mk(ctx, session, max_late_rows=5)
    try:
        a.apply(np.arange(6, dtype=np.uint64), np.arange(6), np.arange(6), np.full(6, A + 50 * S, np.int64))
        _expect(lambda: a.apply(np.arange(6, dtype=np.uint64), np.arange(6) + 20, np.arange(6), np.full(6, A, np.int64)), 3, "max_late_rows")
        _refused(a)
    finally:
        a.close()
    a = _mk(ctx, session, max_emit_rows=10)
    try:
        a.apply(np.arange(11, dtype=np.uint64), np.arange(11), np.arange(11), np.full(11, A, np.int64))
        _expect(a.eof, 3, "max_emit_rows")
    finally:
        a.close()
    if session:  # closed rows and their merged ids share max_emit_rows: 2 closing sessions, 1 merged id
        a = _mk(ctx, True, gap_us=10 * S, wait_us=None, max_emit_rows=2)
        try:
            a.apply(np.array([1, 1, 1, 2], np.uint64), np.arange(4), np.arange(4), np.array([A, A + 20 * S, A + 10 * S, A], np.int64))
            out = a.eof()
            assert out.closed_key.tolist() == [1, 2] and out.merged(0) == [1] and out.merged(1) == []
        finally:
            a.close()


def test_release_buffer_grows_with_held_handles(ctx):
    """Ten calls of 16 rows, each the new pick of its window, held until EOF, which releases them: the release buffer
    (one batch to start with) grows with the handles held."""
    a = _mk(ctx, wait_us=None, length_us=100 * S, max_batch_rows=16)
    try:
        for c in range(10):
            a.apply(np.arange(16, dtype=np.uint64) + 100 * c, np.arange(16) + 16 * c, np.full(16, c), np.full(16, A + c * S, np.int64))
            out = a.advance()
            assert out.closed_key.size == 0 and out.released.size == 0
        out = a.eof()
        assert sorted(out.released.tolist()) == list(range(160)) and out.closed_key.size == 160
    finally:
        a.close()


def test_eof_keeps_sessions_near_utc_max(ctx):
    a = _mk(ctx, True, gap_us=2 * S)
    try:
        a.apply(np.array([1, 2], np.uint64), np.array([0, 1]), np.array([0, 0]), np.array([UTC_MAX - S, UTC_MAX - 3 * S], np.int64))
        out = a.eof()
        assert out.closed_key.tolist() == [2] and out.released.tolist() == [1]
    finally:
        a.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(extreme="sum"), dict(by_dtype="u64"), dict(by_dtype="f32"), dict(length_us=0), dict(offset_us=20 * S),
               dict(gap_us=-1), dict(wait_us=-1), dict(max_windows_per_key=0), dict(max_windows_per_key=65), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as ei:
            gpu.ArgWindow(ctx, **kw)
        assert ei.value.status == 4, kw
    a = _mk(ctx, max_batch_rows=4)
    try:
        _expect(lambda: a.apply(np.arange(5, dtype=np.uint64), np.arange(5), np.arange(5), np.full(5, A, np.int64)), 4, "max_batch_rows")
    finally:
        a.close()
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as ei:
            gpu.ArgWindow(ctxs[0])
        assert ei.value.status == 4 and "one GPU" in str(ei.value)
    finally:
        for c in ctxs:
            c.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle(session):
        a = gpu.ArgWindow(ctx, "max", "f64", 10 * S, 5 * S, A, gap_us=S if session else None, wait_us=S, capacity_hint=1 << 16,
                          max_windows_per_key=16)
        rnd = random.Random(1)
        keys = np.array([rnd.randrange(5000) for _ in range(20000)], np.uint64)
        a.apply(keys, np.arange(keys.size), np.array([rnd.random() for _ in range(keys.size)]), A + np.arange(keys.size, dtype=np.int64) * 1000)
        a.advance(system_now_us=A + 100 * S)
        a.eof()
        a.close()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    for session in (False, True):
        cycle(session)
        before = free()
        for _ in range(3):
            cycle(session)
        assert before - free() < (32 << 20)
