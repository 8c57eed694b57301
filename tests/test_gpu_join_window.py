"""K8: `join_window` on the device (`bw_jwin_*`) against the reference's own join windows.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/join_window_cases.json (made
by the reference's `_WindowLogic` + `_SlidingWindowerLogic` + `_JoinWindowLogic`, tools/gen_join_window_golden.py), the
SHA-256 digests of its seeded streams, and `tests/join_window_oracle.run_join_window` on larger streams -- including the
handles each call releases."""

import json
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import join_window_oracle as jo

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = jo.S, jo.A
SENTINEL = 2**64 - 1


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _join(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    kw.setdefault("max_windows_per_key", 64)
    return gpu.JoinWindow(ctx, spec["insert_mode"], spec["emit_mode"], spec["ordered"], spec["sides"], spec["length_us"],
                          spec["offset_us"], spec["align_us"], None if wait == jo.WAIT_FOREVER else wait, **kw)


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


def _rows(out, bounds, batch):
    """Device rows of one call as the reference's row list.  The device's own order is checked, not restored: per key its
    late rows (arrival order, ids ascending), its down rows (insert-time rows, then one `final` row per closed window
    in the order of its meta rows), its meta rows; the three streams are then interleaved key by key."""
    lk, lw, lr, la = out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist(), out.late_activation.tolist()
    dk, dw, dt = out.down_key.tolist(), out.down_window_id.tolist(), out.tuples()
    mk, mw = out.meta_key.tolist(), out.meta_window_id.tolist()
    gl, gd, gm = _groups(lk, "late"), _groups(dk, "down"), _groups(mk, "meta")
    final = batch is not None and batch.get("final") or False
    rows = []
    for k in sorted(set(gl) | set(gd) | set(gm), key=str):
        for i in gl.get(k, []):
            assert batch is not None and la[i] == batch["act"]
            rows.append([k, lw[i], "L", [batch["sides"][lr[i]], batch["vals"][lr[i]]]])
        di, mi = gd.get(k, []), gm.get(k, [])
        n_close = len(mi) if final else 0
        rows.extend([k, dw[i], "E", list(dt[i])] for i in di[: len(di) - n_close])
        tail = di[len(di) - n_close :]
        for j, i in enumerate(mi):
            if final:
                assert dw[tail[j]] == mw[i], "final row out of meta order"
                rows.append([k, dw[tail[j]], "E", list(dt[tail[j]])])
            rows.append([k, mw[i], "M", list(bounds(mw[i]))])
    return rows


def run_device(ctx, spec, steps, **kw):
    """Drive a JoinWindow through golden-format steps: (rows, sorted released handles) per step, then EOF."""
    j = _join(ctx, spec, **kw)
    final = spec["emit_mode"] == "final"
    acts, released, n_act = [], [], 0

    def take(out, batch):
        acts.append(_rows(out, j.window_bounds, batch))
        released.append(sorted(out.released.tolist()))

    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                _, now, keys, ts, sides, vals = step
                j.apply(np.array(keys, dtype=np.uint64), np.array(sides, dtype=np.uint8), np.array(vals, dtype=np.uint64),
                        np.array(ts, dtype=np.int64), epoch=i + 1, system_now_us=now)
                take(j.advance(), dict(act=n_act, sides=sides, vals=vals, final=final))
                n_act += 1
            else:
                take(j.advance(system_now_us=step[1]), dict(act=None, final=final))
        take(j.eof(), dict(act=None, final=final))
    finally:
        j.close()
    return acts, released


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "join_window_cases.json")


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
    assert released == jo.run_join_window(case["spec"], case["steps"])[1]


@pytest.mark.parametrize("seed", list(jo.SEEDED))
def test_seeded_digests(ctx, golden, seed):
    spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
    got, released = run_device(ctx, spec, steps)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]
    assert released == jo.run_join_window(spec, steps)[1]


def _big_stream(seed, n_act, rows, n_keys, sides, moving=True, hot_rows=0):
    rnd = np.random.default_rng(seed)
    steps, base, now, nxt = [], A, A + 100 * S, 0
    for b in range(n_act):
        keys = rnd.integers(0, n_keys, rows).astype(np.uint64)
        keys[rnd.random(rows) < 0.001] = SENTINEL
        if hot_rows:
            keys[:hot_rows] = 7
        ts = base + rnd.integers(-4 * S, 4 * S, rows) - np.where(rnd.random(rows) < 0.05, rnd.integers(5 * S, 30 * S, rows), 0)
        if moving:
            now += int(rnd.integers(0, 2 * S))
        steps.append(["batch", now, keys.tolist(), ts.tolist(), rnd.integers(0, sides, rows).tolist(), list(range(nxt, nxt + rows))])
        nxt += rows
        if moving and b % 2:  # (`now_getter()` never goes backwards)
            now += 3 * S
            steps.append(["notify", now])
        base += 3 * S
    return steps


COMBOS = [(i, e, o) for i, e in jo.MODES for o in (True, False)]


@pytest.mark.parametrize("ins,emit,ordered", COMBOS)
def test_random_streams_match_oracle(ctx, ins, emit, ordered):
    """About 2^18 rows in six activations over 4000 keys, tumbling or sliding, against the oracle; every input handle is
    released by EOF, and after every call the device holds exactly the handles the oracle holds."""
    k = COMBOS.index((ins, emit, ordered))
    sliding = (k + k // 2) % 2 == 1  # each mode pair: tumbling in one order, sliding in the other
    spec = dict(insert_mode=ins, emit_mode=emit, ordered=ordered, sides=1 + (k // 3) % 4, length_us=4 * S,
                offset_us=2 * S if sliding else 4 * S, align_us=A + 123_457, wait_us=(S, 3 * S)[(k // 4) % 2])
    steps = _big_stream(100 + k, 6, 44_000, 4000, spec["sides"])
    want, want_rel = jo.run_join_window(spec, steps)
    got, rel = run_device(ctx, spec, steps, capacity_hint=1 << 13, max_batch_rows=1 << 16, max_queued_rows=1 << 18)
    assert sum(r[2] == "L" for a in want for r in a) > 1000 and sum(r[2] == "E" for a in want for r in a) > 1000
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"step {i}"
    assert len(got) == len(want)
    assert rel == want_rel
    assert sorted(h for r in rel for h in r) == list(range(sum(len(s[5]) for s in steps if s[0] == "batch")))


def test_hot_key_ordered_wait_forever(ctx):
    """One key with 10^5 queued items (next to 20 000 light keys), ordered, wait forever: nothing is due before EOF, which
    sorts the whole pool into play order."""
    spec = dict(insert_mode="last", emit_mode="running", ordered=True, sides=2, length_us=100 * S, offset_us=100 * S, align_us=A,
                wait_us=jo.WAIT_FOREVER)
    steps = _big_stream(5, 3, 60_000, 20_000, 2, moving=False, hot_rows=35_000)
    assert sum(k == 7 for s in steps for k in s[2]) >= 100_000
    want = jo.run_join_window(spec, steps)
    got = run_device(ctx, spec, steps, capacity_hint=1 << 15, max_batch_rows=1 << 16, max_queued_rows=200_000)
    assert not any(got[0][:-1]) and len(got[0][-1]) > 100_000
    assert got == want


# ---------------------------------------------------------------------------
# capacity and spec edges
# ---------------------------------------------------------------------------


def _expect_capacity(fn, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == 3 and what in str(ei.value), str(ei.value)


def _refused(j):
    with pytest.raises(N.BwError) as ei:
        j.advance()
    assert ei.value.status == 5


def _mk(ctx, **kw):
    from bytewax_b200 import gpu

    args = dict(insert_mode="last", emit_mode="final", ordered=False, sides=2, length_us=10 * S, align_us=A, wait_us=0)
    args.update(kw)
    return gpu.JoinWindow(ctx, **args)


def _ones(n, v=0):
    return np.full(n, v, np.uint8)


@pytest.mark.parametrize("ordered", [False, True])
def test_key_table_exactly_full(ctx, ordered):
    # ordered: the failing call's entries still go through the pool sort and flush, which must stay within the table
    j = _mk(ctx, capacity_hint=16, ordered=ordered)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, SENTINEL], dtype=np.uint64)
        ts = np.full(keys.size, A, np.int64)
        j.apply(keys, _ones(keys.size), np.arange(keys.size), ts)
        out = j.advance()
        assert out.down_key.size == 0 and out.released.size == 0
        j.apply(keys, _ones(keys.size, 1), np.arange(keys.size) + 5000, ts + 10 * S)  # every key closes its first window
        out = j.advance()
        assert out.meta_key.size == 1025 and out.down_key.size == 1025 and sorted(out.released.tolist()) == list(range(1025))
        _expect_capacity(lambda: j.apply(np.array([2000, 2001], np.uint64), _ones(2), np.array([1, 2]), np.array([A, A], np.int64)),
                         "key table full")
        _refused(j)
    finally:
        j.close()


def test_windows_per_key_exactly_full(ctx):
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, length_us=6 * S, offset_us=2 * S, wait_us=None, max_windows_per_key=4)
        try:
            # each item opens 3 windows; two items 2 s apart share two of them: 4 open windows
            j.apply(np.array([3, 3], np.uint64), np.array([0, 1], np.uint8), np.array([1, 2]), np.array([A, A + 2 * S], np.int64))
            if ok:
                out = j.eof()
                assert out.meta_window_id.tolist() == [-2, -1, 0, 1] and sorted(out.released.tolist()) == [1, 2]
            else:
                _expect_capacity(lambda: j.apply(np.array([3], np.uint64), _ones(1), np.array([3]), np.array([A + 4 * S], np.int64)),
                                 "max_windows_per_key")
                _refused(j)
        finally:
            j.close()


def test_queue_pool_exactly_full(ctx):
    j = _mk(ctx, ordered=True, wait_us=None, max_queued_rows=10)
    try:
        j.apply(np.arange(6, dtype=np.uint64), _ones(6), np.arange(6), np.full(6, A, np.int64))
        j.apply(np.arange(4, dtype=np.uint64), _ones(4, 1), np.arange(4) + 6, np.full(4, A + S, np.int64))
        assert j.advance().down_key.size == 0
        _expect_capacity(lambda: j.apply(np.array([9], np.uint64), _ones(1), np.array([10]), np.array([A], np.int64)), "max_queued_rows")
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
        _expect_capacity(lambda: j.apply(np.arange(6, dtype=np.uint64), _ones(6), np.arange(6) + 20, np.full(6, A, np.int64)), "max_late_rows")
    finally:
        j.close()
    j = _mk(ctx, emit_mode="running", max_emit_rows=10)
    try:
        _expect_capacity(lambda: j.apply(np.arange(11, dtype=np.uint64), _ones(11), np.arange(11), np.full(11, A, np.int64)),
                         "max_emit_rows")
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
        with pytest.raises(N.BwError) as ei:
            j.advance()
        assert ei.value.status == 4 and "side" in str(ei.value), str(ei.value)
        _refused(j)
    finally:
        j.close()


def test_release_buffer_grows_with_held_handles(ctx):
    """Ten calls of 16 rows held until EOF, which releases all 160 in one call: the release buffer (one batch to start
    with) grows with the handles held."""
    j = _mk(ctx, ordered=True, wait_us=None, max_batch_rows=16)
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


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(insert_mode="product"), dict(emit_mode="all"), dict(sides=0), dict(sides=5), dict(length_us=0),
               dict(offset_us=0), dict(length_us=S, offset_us=2 * S), dict(wait_us=-1), dict(max_windows_per_key=0),
               dict(max_windows_per_key=65), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as ei:
            gpu.JoinWindow(ctx, **kw)
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
            gpu.JoinWindow(ctxs[0])
        assert ei.value.status == 4 and "one GPU" in str(ei.value)
    finally:
        for c in ctxs:
            c.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle():
        j = gpu.JoinWindow(ctx, "first", "complete", True, 3, S, None, A, S, capacity_hint=1 << 16, max_windows_per_key=16)
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
