"""K10: `join_window` over session windows on the device (`bw_sjwin_*`) against the reference's own session joins.
-m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/session_join_cases.json (made
by the reference's `_WindowLogic` + `_SessionWindowerLogic` + `_JoinWindowLogic`, tools/gen_session_join_golden.py), the
SHA-256 digests of its seeded streams, and `tests/session_join_oracle.run_session_join` on larger streams -- including
the handles each call releases."""

import json
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import session_join_oracle as sj

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = sj.S, sj.A
SENTINEL = 2**64 - 1
UTC_MAX = 253_402_300_799_999_999


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _join(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    kw.setdefault("max_sessions_per_key", 64)
    return gpu.SessionJoinWindow(ctx, spec["insert_mode"], spec["emit_mode"], spec["ordered"], spec["sides"], spec["gap_us"],
                                 None if wait == sj.WAIT_FOREVER else wait, **kw)


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


def _rows(out, batch, final):
    """Device rows of one call as the reference's row list.  The device's own order is checked, not restored: per key its
    late rows (arrival order), its down rows (insert and merge rows, then one `final` row per closed session in the
    order of its meta rows), its meta rows (id order); the three streams are then interleaved key by key."""
    lk, lw, lr, la = out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist(), out.late_activation.tolist()
    dk, dw, dt = out.down_key.tolist(), out.down_window_id.tolist(), out.tuples()
    mk, mw = out.meta_key.tolist(), out.meta_window_id.tolist()
    mo, mc = out.meta_open_us.tolist(), out.meta_close_us.tolist()
    gl, gd, gm = _groups(lk, "late"), _groups(dk, "down"), _groups(mk, "meta")
    rows = []
    for k in sorted(set(gl) | set(gd) | set(gm), key=str):
        for i in gl.get(k, []):
            assert batch is not None and la[i] == batch["act"] and lw[i] == -1
            rows.append([k, -1, "L", [batch["sides"][lr[i]], batch["vals"][lr[i]]]])
        di, mi = gd.get(k, []), gm.get(k, [])
        assert mi == sorted(mi, key=lambda i: mw[i]), "meta rows not in id order"
        n_close = len(mi) if final else 0
        rows.extend([k, dw[i], "E", list(dt[i])] for i in di[: len(di) - n_close])
        tail = di[len(di) - n_close :]
        for j, i in enumerate(mi):
            if final:
                assert dw[tail[j]] == mw[i], "final row out of meta order"
                rows.append([k, dw[tail[j]], "E", list(dt[tail[j]])])
            rows.append([k, mw[i], "M", [mo[i], mc[i], out.merged(i)]])
    return rows


def run_device(ctx, spec, steps, device_cols=False, **kw):
    """Drive a SessionJoinWindow through golden-format steps: (rows, sorted released handles) per step, then EOF."""
    j = _join(ctx, spec, **kw)
    final = spec["emit_mode"] == "final"
    acts, released, n_act = [], [], 0

    def take(out, batch):
        acts.append(_rows(out, batch, final))
        released.append(sorted(out.released.tolist()))

    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                _, now, keys, ts, sides, vals = step
                cols = (np.array(keys, dtype=np.uint64), np.array(sides, dtype=np.uint8), np.array(vals, dtype=np.uint64),
                        np.array(ts, dtype=np.int64))
                if device_cols:
                    d = [torch.from_numpy(c.view(np.int64) if c.dtype == np.uint64 else c).cuda() for c in cols]
                    j.apply_device(*(t.data_ptr() for t in d), len(keys), epoch=i + 1, system_now_us=now)
                    out = j.advance()  # (waits for the call: the columns stay alive until then)
                    del d
                else:
                    j.apply(*cols, epoch=i + 1, system_now_us=now)
                    out = j.advance()
                take(out, dict(act=n_act, sides=sides, vals=vals))
                n_act += 1
            else:
                take(j.advance(system_now_us=step[1]), None)
        take(j.eof(), None)
    finally:
        j.close()
    return acts, released


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "session_join_cases.json")


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
    assert released == sj.run_session_join(case["spec"], case["steps"])[1]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case_other_order(ctx, golden, name):
    """The same steps with `ordered` flipped, against the oracle (which matches every golden case)."""
    case = golden["cases"][name]
    spec = dict(case["spec"], ordered=not case["spec"]["ordered"])
    assert run_device(ctx, spec, case["steps"]) == sj.run_session_join(spec, case["steps"])


@pytest.mark.parametrize("seed", list(sj.SEEDED))
def test_seeded_digests(ctx, golden, seed):
    spec, steps = sj.seeded_steps(seed, moving=seed % 3 != 0)
    got, released = run_device(ctx, spec, steps)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]
    assert released == sj.run_session_join(spec, steps)[1]


def test_apply_device_matches_apply(ctx):
    for seed in (1, 8, 19, 30):
        spec, steps = sj.seeded_steps(seed)
        assert run_device(ctx, spec, steps, device_cols=True) == run_device(ctx, spec, steps)


def _big_stream(seed, n_act, rows, n_keys, sides, moving=True, hot_rows=0, spread=4 * S):
    rnd = np.random.default_rng(seed)
    steps, base, now, nxt = [], A, A + 100 * S, 0
    for b in range(n_act):
        keys = rnd.integers(0, n_keys, rows).astype(np.uint64)
        keys[rnd.random(rows) < 0.001] = SENTINEL
        if hot_rows:
            keys[:hot_rows] = 7
        ts = base + rnd.integers(-spread, spread, rows) - np.where(rnd.random(rows) < 0.05, rnd.integers(5 * S, 30 * S, rows), 0)
        if moving:
            now += int(rnd.integers(0, 2 * S))
        steps.append(["batch", now, keys.tolist(), ts.tolist(), rnd.integers(0, sides, rows).tolist(), list(range(nxt, nxt + rows))])
        nxt += rows
        if moving and b % 2:  # (`now_getter()` never goes backwards)
            now += 3 * S
            steps.append(["notify", now])
        base += 3 * S
    return steps


COMBOS = [(i, e, o) for i, e in sj.MODES for o in (True, False)]


@pytest.mark.parametrize("ins,emit,ordered", COMBOS)
def test_random_streams_match_oracle(ctx, ins, emit, ordered):
    """About 2^16 rows in six activations over 1000 keys with late rows and a moving clock, against the oracle; every
    input handle is released by EOF."""
    k = COMBOS.index((ins, emit, ordered))
    spec = dict(insert_mode=ins, emit_mode=emit, ordered=ordered, sides=1 + (k // 3) % 4, gap_us=(S // 50, S // 5)[k % 2],
                wait_us=(S, 3 * S)[(k // 4) % 2])
    steps = _big_stream(100 + k, 6, 11_000, 1000, spec["sides"])
    stats = {}
    want, want_rel = sj.run_session_join(spec, steps, stats=stats)
    got, rel = run_device(ctx, spec, steps, capacity_hint=1 << 11, max_batch_rows=1 << 14, max_queued_rows=1 << 17)
    assert sum(r[2] == "L" for a in want for r in a) > 1000 and sum(r[2] == "M" for a in want for r in a) > 1000
    assert ordered or stats["merges"] > 20
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"step {i}"
    assert len(got) == len(want)
    assert rel == want_rel
    assert sorted(h for r in rel for h in r) == list(range(sum(len(s[5]) for s in steps if s[0] == "batch")))


def test_hot_key_unordered_one_long_session(ctx):
    """10^5 items of one key per activation, all within the gap of each other: one session, walked by one thread."""
    spec = dict(insert_mode="last", emit_mode="running", ordered=False, sides=2, gap_us=10 * S, wait_us=5 * S)
    steps = _big_stream(6, 2, 120_000, 5000, 2, moving=False, hot_rows=100_000, spread=2 * S)
    want = sj.run_session_join(spec, steps)
    got = run_device(ctx, spec, steps, capacity_hint=1 << 13, max_batch_rows=1 << 17, max_emit_rows=1 << 19)
    assert sum(r[0] == 7 and r[2] == "E" for a in want[0] for r in a) >= 180_000
    assert sum(r[0] == 7 and r[2] == "M" for a in want[0] for r in a) == 1
    assert got == want


def test_hot_key_ordered_wait_forever(ctx):
    """One key with 10^5 queued items (next to 5000 light keys), ordered, wait forever: nothing is due before EOF, which
    sorts the whole pool into play order."""
    spec = dict(insert_mode="first", emit_mode="running", ordered=True, sides=2, gap_us=10 * S, wait_us=sj.WAIT_FOREVER)
    steps = _big_stream(5, 3, 60_000, 5000, 2, moving=False, hot_rows=35_000)
    assert sum(k == 7 for s in steps for k in s[2]) >= 100_000
    want = sj.run_session_join(spec, steps)
    got = run_device(ctx, spec, steps, capacity_hint=1 << 13, max_batch_rows=1 << 16, max_queued_rows=200_000)
    assert not any(got[0][:-1]) and len(got[0][-1]) > 100_000
    assert got == want


# ---------------------------------------------------------------------------
# capacity and spec edges
# ---------------------------------------------------------------------------


def _expect(fn, status, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == status and what in str(ei.value), str(ei.value)


def _refused(j):
    with pytest.raises(N.BwError) as ei:
        j.advance()
    assert ei.value.status == 5


def _mk(ctx, **kw):
    from bytewax_b200 import gpu

    args = dict(insert_mode="last", emit_mode="final", ordered=False, sides=2, gap_us=S, wait_us=0)
    args.update(kw)
    return gpu.SessionJoinWindow(ctx, **args)


def _ones(n, v=0):
    return np.full(n, v, np.uint8)


@pytest.mark.parametrize("ordered", [False, True])
def test_key_table_exactly_full(ctx, ordered):
    j = _mk(ctx, capacity_hint=16, ordered=ordered)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, SENTINEL], dtype=np.uint64)
        ts = np.full(keys.size, A, np.int64)
        j.apply(keys, _ones(keys.size), np.arange(keys.size), ts)
        out = j.advance()
        assert out.down_key.size == 0 and out.released.size == 0
        j.apply(keys, _ones(keys.size, 1), np.arange(keys.size) + 5000, ts + 10 * S)  # every key closes its first session
        out = j.advance()
        assert out.meta_key.size == 1025 and out.down_key.size == 1025 and sorted(out.released.tolist()) == list(range(1025))
        _expect(lambda: j.apply(np.array([2000, 2001], np.uint64), _ones(2), np.array([1, 2]), np.array([A, A], np.int64)), 3,
                "key table full")
        _refused(j)
    finally:
        j.close()


def test_sessions_per_key_exactly_full(ctx):
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, gap_us=0, wait_us=None, max_sessions_per_key=4)
        try:
            n = 4 + extra
            call = lambda: j.apply(np.full(n, 3, np.uint64), _ones(n), np.arange(n), A + np.arange(n, dtype=np.int64) * S)  # noqa: E731
            if ok:
                call()
                out = j.eof()
                assert out.meta_window_id.tolist() == [0, 1, 2, 3] and sorted(out.released.tolist()) == [0, 1, 2, 3]
            else:
                _expect(call, 3, "max_sessions_per_key")
                _refused(j)
        finally:
            j.close()


def test_merged_ids_exactly_full(ctx):
    """M = 3: a survivor holds 3 merged ids; a fourth merge into it fails."""
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, gap_us=10 * S, wait_us=None, max_sessions_per_key=3)
        try:
            def one(a, b, h):  # a new session at a, then b extends session 0 to within gap of it: one merge per call
                j.apply(np.array([5, 5], np.uint64), _ones(2), np.array([h, h + 1]), np.array([a, b], np.int64))

            one(A, A, 0)
            for c in range(3):
                one(A + (20 + 20 * c) * S, A + (10 + 20 * c) * S, 2 * c + 2)
            assert j.advance().meta_key.size == 0
            if ok:
                out = j.eof()
                assert out.meta_window_id.tolist() == [0] and out.merged(0) == [1, 2, 3]
                assert [out.meta_open_us[0], out.meta_close_us[0]] == [A, A + 60 * S]
            else:
                _expect(lambda: one(A + 80 * S, A + 70 * S, 10), 3, "merged ids")
                _refused(j)
        finally:
            j.close()


def test_queue_pool_exactly_full(ctx):
    j = _mk(ctx, ordered=True, wait_us=None, max_queued_rows=10)
    try:
        j.apply(np.arange(6, dtype=np.uint64), _ones(6), np.arange(6), np.full(6, A, np.int64))
        j.apply(np.arange(4, dtype=np.uint64), _ones(4, 1), np.arange(4) + 6, np.full(4, A + S, np.int64))
        assert j.advance().down_key.size == 0
        _expect(lambda: j.apply(np.array([9], np.uint64), _ones(1), np.array([10]), np.array([A], np.int64)), 3, "max_queued_rows")
        _refused(j)
    finally:
        j.close()
    j = _mk(ctx, ordered=True, wait_us=None, max_queued_rows=10)
    try:
        j.apply(np.arange(10, dtype=np.uint64), _ones(10), np.arange(10), np.full(10, A, np.int64))
        out = j.eof()
        assert out.down_key.size == 10 and sorted(out.released.tolist()) == list(range(10))
    finally:
        j.close()


def test_emit_and_late_buffers_exactly_full(ctx):
    j = _mk(ctx, emit_mode="running", max_emit_rows=10, max_late_rows=5)
    try:
        j.apply(np.arange(10, dtype=np.uint64), _ones(10), np.arange(10), np.full(10, A + 5 * S, np.int64))  # 10 running rows
        j.apply(np.arange(5, dtype=np.uint64), _ones(5), np.arange(5) + 10, np.full(5, A, np.int64))  # 5 lates
        out = j.advance()
        assert out.down_key.size == 10 and out.late_key.size == 5 and out.late_row.tolist() == list(range(5))
        assert sorted(out.released.tolist()) == list(range(10, 15))
        _expect(lambda: j.apply(np.arange(6, dtype=np.uint64), _ones(6), np.arange(6) + 20, np.full(6, A, np.int64)), 3, "max_late_rows")
    finally:
        j.close()
    j = _mk(ctx, emit_mode="running", max_emit_rows=10)
    try:
        _expect(lambda: j.apply(np.arange(11, dtype=np.uint64), _ones(11), np.arange(11), np.full(11, A, np.int64)), 3, "max_emit_rows")
    finally:
        j.close()
    # meta rows and their merged ids share max_emit_rows: 2 closing sessions, 1 merged id
    j = _mk(ctx, emit_mode="complete", gap_us=10 * S, wait_us=None, max_emit_rows=2)
    try:
        j.apply(np.array([1, 1, 1, 2], np.uint64), _ones(4), np.arange(4), np.array([A, A + 20 * S, A + 10 * S, A], np.int64))
        out = j.eof()
        assert out.meta_key.tolist() == [1, 2] and out.merged(0) == [1] and out.merged(1) == []
    finally:
        j.close()


@pytest.mark.parametrize("ordered", [False, True])
def test_device_side_out_of_range(ctx, ordered):
    """Device columns are not checked on the host: a side >= sides is not played, and the join reports it and stops."""
    j = _mk(ctx, sides=2, ordered=ordered)
    try:
        d = lambda a, dt: torch.tensor(a, dtype=dt, device="cuda")  # noqa: E731
        keys, sides = d([1, 2, 3], torch.int64), d([0, 4, 1], torch.uint8)
        hs, ts = d([10, 11, 12], torch.int64), d([A, A, A], torch.int64)
        j.apply_device(keys.data_ptr(), sides.data_ptr(), hs.data_ptr(), ts.data_ptr(), 3)
        _expect(j.advance, 4, "side")
        _refused(j)
    finally:
        j.close()


def test_release_buffer_grows_with_held_handles(ctx):
    """Ten calls of 16 rows held until EOF, which releases all 160 in one call: the release buffer (one batch to start
    with) grows with the handles held."""
    j = _mk(ctx, ordered=True, wait_us=None, gap_us=10 * S, max_batch_rows=16)
    try:
        for c in range(10):
            j.apply(np.arange(16, dtype=np.uint64) + 100 * (c % 2), _ones(16, c % 2), np.arange(16) + 16 * c,
                    np.full(16, A + c * S, np.int64))
            out = j.advance()
            assert out.down_key.size == 0 and out.released.size == 0
        out = j.eof()
        assert sorted(out.released.tolist()) == list(range(160)) and out.meta_key.size == 32
    finally:
        j.close()


def test_eof_keeps_sessions_near_utc_max(ctx):
    j = _mk(ctx, gap_us=2 * S)
    try:
        j.apply(np.array([1, 2], np.uint64), _ones(2), np.array([0, 1]), np.array([UTC_MAX - S, UTC_MAX - 3 * S], np.int64))
        out = j.eof()
        assert out.meta_key.tolist() == [2] and out.released.tolist() == [1]
    finally:
        j.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(insert_mode="product"), dict(emit_mode="all"), dict(sides=0), dict(sides=5), dict(gap_us=-1), dict(wait_us=-1),
               dict(max_sessions_per_key=0), dict(max_sessions_per_key=65), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as ei:
            gpu.SessionJoinWindow(ctx, **kw)
        assert ei.value.status == 4, kw
    j = _mk(ctx, sides=2)
    try:
        with pytest.raises(N.BwError) as ei:
            j.apply(np.array([1], np.uint64), np.array([2], np.uint8), np.array([1]), np.array([A], np.int64))
        assert ei.value.status == 4
    finally:
        j.close()
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as ei:
            gpu.SessionJoinWindow(ctxs[0])
        assert ei.value.status == 4 and "one GPU" in str(ei.value)
    finally:
        for c in ctxs:
            c.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle():
        j = gpu.SessionJoinWindow(ctx, "first", "complete", True, 3, S, S, capacity_hint=1 << 16, max_sessions_per_key=16)
        rnd = random.Random(1)
        keys = np.array([rnd.randrange(5000) for _ in range(20000)], np.uint64)
        j.apply(keys, np.array([rnd.randrange(3) for _ in range(keys.size)], np.uint8), np.arange(keys.size),
                A + np.arange(keys.size, dtype=np.int64) * 1000)
        j.advance(system_now_us=A + 100 * S)
        j.eof()
        j.close()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    cycle()
    before = free()
    for _ in range(3):
        cycle()
    assert before - free() < (32 << 20)
