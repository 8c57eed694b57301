"""K9: `collect_window` on the device (`bw_collect_*`) against the reference's own collect windows.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/collect_window_cases.json
(made by the reference's `_WindowLogic` + `_SlidingWindowerLogic` + `_FoldWindowLogic` with the collect callbacks,
tools/gen_collect_window_golden.py), the SHA-256 digests of its seeded streams, and
`tests/collect_window_oracle.run_collect_window` on larger streams -- with the handles each call releases."""

import json
import os

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import collect_window_oracle as co

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = co.S, co.A
SENTINEL = 2**64 - 1


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _collect(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    kw.setdefault("max_windows_per_key", 64)
    return gpu.CollectWindow(ctx, spec["ordered"], spec["length_us"], spec["offset_us"], spec["align_us"],
                             None if wait == co.WAIT_FOREVER else wait, **kw)


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


def _rows(out, bounds, batch, handle_of=None):
    """Device rows of one call as the reference's row list: per key its late rows (arrival order, ids ascending), then
    per closed window its list and its metadata row.  ``handle_of`` maps a handle back to the golden value."""
    hv = handle_of or (lambda h: h)
    lk, lw, lr, la = out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist(), out.late_activation.tolist()
    dk, dw, lists = out.down_key.tolist(), out.down_window_id.tolist(), out.lists()
    assert out.down_offset[0] == 0 and out.handle.size == out.down_offset[-1]
    gl, gd = _groups(lk, "late"), _groups(dk, "down")
    rows = []
    for k in sorted(set(gl) | set(gd), key=str):
        for i in gl.get(k, []):
            assert batch is not None and la[i] == batch["act"]
            rows.append([k, lw[i], "L", batch["vals"][lr[i]]])
        for i in gd.get(k, []):
            rows.append([k, dw[i], "E", [hv(h) for h in lists[i]]])
            rows.append([k, dw[i], "M", list(bounds(dw[i]))])
    return rows


def run_device(ctx, spec, steps, handle_of=None, handles=None, **kw):
    """Drive a CollectWindow through golden-format steps: (rows, sorted released handles) per step, then EOF.
    ``handles``: the handle to pass for each golden value (default: the value itself)."""
    c = _collect(ctx, spec, **kw)
    acts, released, n_act = [], [], 0
    hmap = handles or (lambda v: v)

    def take(out, batch):
        acts.append(_rows(out, c.window_bounds, batch, handle_of))
        released.append(sorted(handle_of(h) if handle_of else h for h in out.released.tolist()))

    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                _, now, keys, ts, _sides, vals = step
                c.apply(np.array(keys, dtype=np.uint64), np.array([hmap(v) for v in vals], dtype=np.uint64), np.array(ts, dtype=np.int64),
                        epoch=i + 1, system_now_us=now)
                take(c.advance(), dict(act=n_act, vals=vals))
                n_act += 1
            else:
                take(c.advance(system_now_us=step[1]), dict(act=None))
        take(c.eof(), dict(act=None))
    finally:
        c.close()
    return acts, released


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "collect_window_cases.json")


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
    assert released == co.run_collect_window(case["spec"], case["steps"])[1]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case_other_order(ctx, golden, name):
    """The same steps in the other order, against the oracle (the golden holds the reference's rows in one order)."""
    case = golden["cases"][name]
    spec = dict(case["spec"], ordered=not case["spec"]["ordered"])
    want = co.run_collect_window(spec, case["steps"])
    assert run_device(ctx, spec, case["steps"]) == want


@pytest.mark.parametrize("seed", list(co.SEEDED))
def test_seeded_digests(ctx, golden, seed):
    spec, steps = co.seeded_steps(seed, moving=seed % 3 != 0)
    got, released = run_device(ctx, spec, steps)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]
    assert released == co.run_collect_window(spec, steps)[1]


@pytest.mark.parametrize("name", ["sliding_indivisible_offset", "ordered_ties_stable", "discard_resets_watermark", "near_utc_max"])
def test_any_u64_is_a_handle(ctx, golden, name):
    """Handles 0, 2^64-1 and random bit patterns: no value is reserved."""
    case = golden["cases"][name]
    n = sum(len(s[5]) for s in case["steps"] if s[0] == "batch")
    rnd = np.random.default_rng(3)
    pats = [0, SENTINEL] + [int(x) for x in rnd.integers(0, 2**63, n, dtype=np.uint64) * 2 + 1]
    fwd = {v: pats[v] for v in range(n)}
    back = {h: v for v, h in fwd.items()}
    got, released = run_device(ctx, case["spec"], case["steps"], handle_of=back.__getitem__, handles=fwd.__getitem__)
    assert got == case["acts"]
    assert released == co.run_collect_window(case["spec"], case["steps"])[1]


def _big_stream(seed, n_act, rows, n_keys, moving=True, hot_rows=0):
    rnd = np.random.default_rng(seed)
    steps, base, now, nxt = [], A, A + 100 * S, 0
    for b in range(n_act):
        keys = rnd.integers(0, n_keys, rows).astype(np.uint64)
        keys[rnd.random(rows) < 0.001] = SENTINEL
        if hot_rows:
            keys[:hot_rows] = 7
        ts = base + rnd.integers(-8 * S, 8 * S, rows) - np.where(rnd.random(rows) < 0.05, rnd.integers(10 * S, 90 * S, rows), 0)
        if moving:
            now += int(rnd.integers(0, 2 * S))
        steps.append(["batch", now, keys.tolist(), ts.tolist(), [0] * rows, list(range(nxt, nxt + rows))])
        nxt += rows
        if moving and b % 2:  # (`now_getter()` never goes backwards)
            now += 3 * S
            steps.append(["notify", now])
        base += 6 * S
    return steps


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("shape", ["sliding", "tumbling"])
def test_random_streams_match_oracle(ctx, ordered, shape):
    """About 2^17 rows in eight activations over 1000 keys (sliding 60 s / 10 s or tumbling 10 s), jitter that makes
    rows late and a moving clock, against the oracle; every handle is released once, in the call the rule names."""
    spec = dict(ordered=ordered, length_us=60 * S if shape == "sliding" else 10 * S, offset_us=10 * S, align_us=A + 123_457,
                wait_us=5 * S)
    steps = _big_stream(11 + ordered + 2 * (shape == "sliding"), 8, 16_000, 1000)
    want, want_rel = co.run_collect_window(spec, steps)
    got, rel = run_device(ctx, spec, steps, capacity_hint=1 << 11, max_batch_rows=1 << 14, max_queued_rows=1 << 18)
    assert sum(r[2] == "L" for a in want for r in a) > 1000 and sum(r[2] == "E" for a in want for r in a) > 1000
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"step {i}"
    assert len(got) == len(want)
    assert rel == want_rel
    assert sorted(h for r in rel for h in r) == list(range(sum(len(s[5]) for s in steps if s[0] == "batch")))


@pytest.mark.parametrize("length", [10, 60])
def test_hot_key_one_window(ctx, length):
    """10^6 values of one key, ordered, wait forever, flushed at EOF: one tumbling window holding all of them, or (sliding
    60 s / 10 s) the same values in six windows -- every list materialised in play order."""
    n = 1_000_000
    rnd = np.random.default_rng(5)
    ts = A + 60 * S + rnd.integers(0, 10 * S, n)
    spec = dict(ordered=True, length_us=length * S, offset_us=10 * S, align_us=A, wait_us=co.WAIT_FOREVER)
    c = _collect(ctx, spec, capacity_hint=16, max_batch_rows=1 << 18, max_queued_rows=n)
    try:
        for b in range(0, n, 1 << 18):
            c.apply(np.full(min(1 << 18, n - b), 7, np.uint64), np.arange(b, min(b + (1 << 18), n)), ts[b:b + (1 << 18)])
            out = c.advance()
            assert out.down_key.size == 0 and out.released.size == 0
        out = c.eof()
        want = np.argsort(ts, kind="stable").tolist()
        lists = out.lists()
        assert len(lists) == length // 10 and all(lst == want for lst in lists)
        assert sorted(out.released.tolist()) == list(range(n))
    finally:
        c.close()


def test_entry_store_growth(ctx):
    """Held entries pass the store's starting size (one batch) many times over: the rows equal those of a store sized
    up front, and the oracle's."""
    spec = dict(ordered=False, length_us=60 * S, offset_us=10 * S, align_us=A, wait_us=co.WAIT_FOREVER)
    steps = _big_stream(21, 12, 1000, 50, moving=False)
    want = co.run_collect_window(spec, steps)
    small = run_device(ctx, spec, steps, capacity_hint=64, max_batch_rows=1000)
    large = run_device(ctx, spec, steps, capacity_hint=64, max_batch_rows=1 << 16)
    assert small == large == want
    assert not any(a for a in want[0][:-1] if any(r[2] == "E" for r in a))  # everything held until EOF: 72 000 entries


@pytest.mark.parametrize("ordered", [True, False])
def test_apply_device_equals_apply(ctx, ordered):
    spec = dict(ordered=ordered, length_us=60 * S, offset_us=10 * S, align_us=A, wait_us=2 * S)
    steps = _big_stream(31, 6, 20_000, 500)
    want = run_device(ctx, spec, steps, capacity_hint=1 << 10, max_batch_rows=1 << 15)
    c = _collect(ctx, spec, capacity_hint=1 << 10, max_batch_rows=1 << 15)
    acts, released, n_act = [], [], 0
    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                _, now, keys, ts, _s, vals = step
                d = lambda a: torch.tensor(np.array(a, dtype=np.uint64).view(np.int64), device="cuda")  # noqa: E731
                dk, dh, dt = d(keys), d(vals), torch.tensor(ts, dtype=torch.int64, device="cuda")
                c.apply_device(dk.data_ptr(), dh.data_ptr(), dt.data_ptr(), len(keys), epoch=i + 1, system_now_us=now)
                out = c.advance()
                acts.append(_rows(out, c.window_bounds, dict(act=n_act, vals=vals)))
                n_act += 1
            else:
                out = c.advance(system_now_us=step[1])
                acts.append(_rows(out, c.window_bounds, None))
            released.append(sorted(out.released.tolist()))
        out = c.eof()
        acts.append(_rows(out, c.window_bounds, None))
        released.append(sorted(out.released.tolist()))
    finally:
        c.close()
    assert (acts, released) == want


# ---------------------------------------------------------------------------
# capacity and spec edges
# ---------------------------------------------------------------------------


def _expect_capacity(fn, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == 3 and what in str(ei.value), str(ei.value)


def _refused(c):
    with pytest.raises(N.BwError) as ei:
        c.advance()
    assert ei.value.status == 5


def _mk(ctx, **kw):
    from bytewax_b200 import gpu

    args = dict(ordered=False, length_us=10 * S, align_us=A, wait_us=0)
    args.update(kw)
    return gpu.CollectWindow(ctx, **args)


@pytest.mark.parametrize("ordered", [False, True])
def test_key_table_exactly_full(ctx, ordered):
    c = _mk(ctx, capacity_hint=16, ordered=ordered)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, SENTINEL], dtype=np.uint64)
        ts = np.full(keys.size, A, np.int64)
        c.apply(keys, np.arange(keys.size), ts)
        assert c.advance().down_key.size == 0
        c.apply(keys, np.arange(keys.size) + 5000, ts + 10 * S)  # every key closes its first window
        out = c.advance()
        assert out.down_key.size == 1025 and sorted(out.released.tolist()) == list(range(1025))
        assert all(lst == [i] for i, lst in sorted(zip(out.handle.tolist(), out.lists())))
        _expect_capacity(lambda: c.apply(np.array([2000, 2001], np.uint64), np.array([1, 2]), np.array([A, A], np.int64)), "key table full")
        _refused(c)
    finally:
        c.close()


def test_windows_per_key_exactly_full(ctx):
    for extra, ok in ((0, True), (1, False)):
        c = _mk(ctx, length_us=6 * S, offset_us=2 * S, wait_us=None, max_windows_per_key=4)
        try:
            c.apply(np.array([3, 3], np.uint64), np.array([1, 2]), np.array([A, A + 2 * S], np.int64))  # 4 open windows
            if ok:
                out = c.eof()
                assert out.down_window_id.tolist() == [-2, -1, 0, 1] and out.lists() == [[1], [1, 2], [1, 2], [2]]
                assert sorted(out.released.tolist()) == [1, 2]
            else:
                _expect_capacity(lambda: c.apply(np.array([3], np.uint64), np.array([3]), np.array([A + 4 * S], np.int64)),
                                 "max_windows_per_key")
                _refused(c)
        finally:
            c.close()


def test_queue_exactly_full(ctx):
    c = _mk(ctx, ordered=True, wait_us=None, max_queued_rows=10)
    try:
        c.apply(np.arange(6, dtype=np.uint64), np.arange(6), np.full(6, A, np.int64))
        c.apply(np.arange(4, dtype=np.uint64), np.arange(4) + 6, np.full(4, A + S, np.int64))
        assert c.advance().down_key.size == 0
        _expect_capacity(lambda: c.apply(np.array([9], np.uint64), np.array([10]), np.array([A], np.int64)), "max_queued_rows")
        _refused(c)
    finally:
        c.close()
    c = _mk(ctx, ordered=True, wait_us=None, max_queued_rows=10)
    try:
        c.apply(np.arange(10, dtype=np.uint64), np.arange(10), np.full(10, A, np.int64))
        out = c.eof()
        assert out.down_key.size == 10 and sorted(out.released.tolist()) == list(range(10))
    finally:
        c.close()


def test_late_and_closed_buffers_exactly_full(ctx):
    c = _mk(ctx, max_emit_rows=10, max_late_rows=5)
    try:
        c.apply(np.arange(10, dtype=np.uint64), np.arange(10), np.full(10, A + 5 * S, np.int64))
        c.apply(np.arange(10, dtype=np.uint64), np.arange(10) + 10, np.full(10, A + 15 * S, np.int64))  # 10 windows close
        c.apply(np.arange(5, dtype=np.uint64), np.arange(5) + 20, np.full(5, A, np.int64))  # 5 lates
        out = c.advance()
        assert out.down_key.size == 10 and out.late_key.size == 5 and out.late_row.tolist() == list(range(5))
        assert sorted(out.released.tolist()) == list(range(10)) + list(range(20, 25))
        _expect_capacity(lambda: c.apply(np.arange(6, dtype=np.uint64), np.arange(6) + 30, np.full(6, A, np.int64)), "max_late_rows")
        _refused(c)
    finally:
        c.close()
    c = _mk(ctx, max_emit_rows=10)
    try:
        c.apply(np.arange(11, dtype=np.uint64), np.arange(11), np.full(11, A, np.int64))
        _expect_capacity(lambda: c.apply(np.arange(11, dtype=np.uint64), np.arange(11) + 20, np.full(11, A + 10 * S, np.int64)),
                         "max_emit_rows")
        _refused(c)
    finally:
        c.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(length_us=0), dict(offset_us=0), dict(length_us=S, offset_us=2 * S), dict(wait_us=-1), dict(max_windows_per_key=0),
               dict(max_windows_per_key=65), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as ei:
            gpu.CollectWindow(ctx, **kw)
        assert ei.value.status == 4, kw
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as ei:
            gpu.CollectWindow(ctxs[0])
        assert ei.value.status == 4 and "one GPU" in str(ei.value)
    finally:
        for x in ctxs:
            x.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle():
        c = gpu.CollectWindow(ctx, True, 6 * S, 2 * S, A, S, capacity_hint=1 << 16, max_windows_per_key=16, max_batch_rows=4096)
        rnd = np.random.default_rng(1)
        for b in range(5):  # the store and staging buffers grow past their starting size
            keys = rnd.integers(0, 50, 4096).astype(np.uint64)
            c.apply(keys, np.arange(4096) + 4096 * b, A + np.arange(4096, dtype=np.int64) * 1000)
            c.advance()
        c.advance(system_now_us=A + 100 * S)
        c.eof()
        c.close()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    cycle()
    before = free()
    for _ in range(3):
        cycle()
    assert before - free() < (32 << 20)
