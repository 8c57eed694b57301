"""K12 on the GPU: `collect_window` over session windows (``bw_scwin``) against the restatement in
``tests/session_collect_oracle.py`` -- every row, every list in flattened play order, every merge interval, every
merged id, and the handles each call releases."""

import json
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import session_collect_oracle as sc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = sc.S, sc.A
UTC_MAX = 253_402_300_799_999_999
F = sc.WAIT_FOREVER


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _mk(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    kw.setdefault("max_sessions_per_key", 64)
    return gpu.SessionCollectWindow(ctx, spec["ordered"], spec["gap_us"], None if wait == F else wait, **kw)


def _device_rows(out, hs_in):
    """One call's device rows as the oracle's, per stream (E, M, L), and its released handles, sorted."""
    E, M = [], []
    lists = out.lists()
    for i, (k, w) in enumerate(zip(out.down_key.tolist(), out.down_window_id.tolist())):
        E.append([k, w, "E", [lists[i], [list(x) for x in out.merges(i)]]])
        M.append([k, w, "M", [int(out.open_us[i]), int(out.close_us[i]), out.merged(i)]])
    L = [[k, -1, "L", int(hs_in[r])] for k, r in zip(out.late_key.tolist(), out.late_row.tolist())]
    return E, M, L, sorted(out.released.tolist())


def run_device(ctx, spec, steps, device_cols=False, **kw):
    """Per step, then EOF: (E rows, M rows, L rows, released) from the device."""
    j = _mk(ctx, spec, **kw)
    res = []
    try:
        for step in steps:
            if step[0] == "batch":
                keys, ts, hs = np.array(step[2], np.uint64), np.array(step[3], np.int64), np.array(step[4], np.uint64)
                if device_cols:
                    d = [torch.from_numpy(a.view(np.int64)).cuda() for a in (keys, hs, ts)]
                    j.apply_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), keys.size, system_now_us=step[1])
                    out = j.advance()
                    del d
                else:
                    j.apply(keys, hs, ts, system_now_us=step[1])
                    out = j.advance()
                res.append(_device_rows(out, hs))
            else:
                res.append(_device_rows(j.advance(system_now_us=step[1]), []))
        res.append(_device_rows(j.eof(), []))
    finally:
        j.close()
    return res


def run_oracle(spec, steps, stats=None):
    acts, rel = sc.run_session_collect(spec, steps, stats=stats)
    out = []
    for rows, r in zip(acts, rel):
        E = [x for x in rows if x[2] == "E"]
        M = [x for x in rows if x[2] == "M"]
        L = [x for x in rows if x[2] == "L"]
        out.append((E, M, L, r))
    return out


def _check(ctx, spec, steps, **kw):
    st = {}
    want = run_oracle(spec, steps, st)
    got = run_device(ctx, spec, steps, **kw)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, g, w)
    assert len(got) == len(want)
    return st["merges"]


class Steps:
    """Hand-built steps; every value is a fresh int (its handle)."""

    def __init__(self, now=A + 10**6 * S):
        self.steps, self.n, self.now = [], 0, now

    def batch(self, *items, now=None):  # items: (key, ts)
        if now is not None:
            self.now = now
        self.steps.append(["batch", self.now, [k for k, _ in items], [t for _, t in items], list(range(self.n, self.n + len(items)))])
        self.n += len(items)
        return self

    def notify(self, now):
        self.now = now
        self.steps.append(["notify", now])
        return self


def spec_(ordered=False, gap=10 * S, wait=F):
    return dict(ordered=ordered, gap_us=gap, wait_us=wait)


# each case: (spec, steps, whether it merges)
CASES = {
    "open_extend_before_after": (spec_(), Steps().batch((1, A + 5 * S), (1, A), (1, A + 12 * S)), False),
    "bridge_merges_two": (spec_(), Steps().batch((1, A), (1, A + 20 * S), (1, A + 21 * S), (1, A + 10 * S)), True),
    # C -> B -> A in one flush: 2 absorbs... the bridge at A+30 merges 2 into 1, the one at A+10 then 1 into 0
    "chain_one_flush": (spec_(), Steps().batch((1, A), (1, A + 1), (1, A + 20 * S), (1, A + 40 * S), (1, A + 41 * S), (1, A + 30 * S),
                                               (1, A + 10 * S), (1, A + 2)), True),
    "merge_across_flushes": (spec_(), Steps().batch((2, A), (2, A + 1), (2, A + 20 * S), (2, A + 20 * S + 1))
                             .batch((2, A + 10 * S), (2, A + 3)).batch((2, A + 25 * S), (2, A + 4)), True),
    "value_in_merged_away_session": (spec_(), Steps().batch((4, A + 20 * S), (4, A), (4, A + 10 * S), (4, A + 11 * S)), True),
    "gap_zero_equal_ts": (spec_(gap=0, wait=0), Steps().batch((1, A), (1, A), (1, A + 1)).batch((1, A + 1), (1, A + 5)), False),
    "late_rows": (spec_(gap=S, wait=0), Steps().batch((3, A + 10 * S), (3, A), (5, A + 10 * S)).batch((3, A + 2 * S), (5, A + 30 * S)), False),
    "moving_clock_notify": (spec_(ordered=False, gap=2 * S, wait=S), Steps(now=A).batch((7, A), (8, A + S), now=A)
                            .notify(A + 2 * S).notify(A + 4 * S).batch((7, A + 5 * S), now=A + 6 * S).notify(A + 20 * S), False),
    "ordered_notify_wakes_queue_head": (spec_(ordered=True, gap=20 * S, wait=10 * S),
                                        Steps(now=A).batch((4, A + 8 * S), (4, A + 5 * S), (4, A + 12 * S), now=A)
                                        .notify(A + 4 * S).notify(A + 6 * S).notify(A + 8 * S).notify(A + 60 * S), False),
    "wait_forever_flush_at_eof": (spec_(ordered=True, gap=S, wait=F),
                                  Steps().batch((1, A + 9 * S), (1, A + S), (1, A + 5 * S)).batch((1, A), (2, A + 3 * S)), False),
    "eof_near_utc_max": (spec_(ordered=True, gap=2 * S, wait=0),
                         Steps().batch((9, UTC_MAX - S), (10, UTC_MAX - 3 * S), (11, UTC_MAX - 2 * S)), False),
}


@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_case(ctx, name, ordered):
    spec, st, merges = CASES[name]
    spec = dict(spec, ordered=ordered)
    n = _check(ctx, spec, st.steps)
    if merges and not ordered:
        assert n > 0, name  # a case named for a merge merges
    if ordered:
        assert n == 0  # ordered mode never merges


@pytest.mark.parametrize("seed", list(sc.SEEDED))
def test_seeded(ctx, seed):
    spec, steps = sc.seeded_steps(seed, moving=seed % 3 != 0)
    n = _check(ctx, spec, steps)
    assert not (spec["ordered"] and n)


# ---- the reference's own rows (tests/golden/session_collect_cases.json, tools/gen_session_collect_golden.py) ----------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "session_collect_cases.json")
with open(GOLDEN) as _f:
    _G = json.load(_f)


def _golden_device(ctx, spec, steps, into):
    """The device's rows as the reference's golden rows: each container built from the device's handles and merge
    intervals with the reference's folder and merger; streams interleaved as the reference's logic returns them (per
    key in ascending key-string order, its late rows, then each closed session's E row and M row)."""
    vo = sc.value_fn(into)
    acts = []
    for E, M, L, _rel in run_device(ctx, spec, steps):
        by = {}
        for r in L:
            by.setdefault(r[0], [[], []])[0].append([r[0], r[1], "L", sc._json(vo(r[3]))])
        for e, m in zip(E, M):
            assert e[:2] == m[:2]
            c = sc.container_json(sc.container(into, e[3][0], e[3][1], vo))
            by.setdefault(e[0], [[], []])[1].extend([[e[0], e[1], "E", c], m])
        acts.append([r for k in sorted(by, key=str) for r in by[k][0] + by[k][1]])
    return acts


@pytest.mark.parametrize("name", sorted(_G["cases"]))
def test_golden_case(ctx, name):
    c = _G["cases"][name]
    assert _golden_device(ctx, c["spec"], c["steps"], c["into"]) == c["acts"]


@pytest.mark.parametrize("name", sorted(_G["cases"]))
def test_golden_case_other_order(ctx, name):
    """The same steps in the other order, against the restatement (which the goldens pin)."""
    c = _G["cases"][name]
    spec = dict(c["spec"], ordered=not c["spec"]["ordered"])
    acts, _ = sc.run_session_collect(spec, c["steps"])
    assert _golden_device(ctx, spec, c["steps"], c["into"]) == sc.golden_rows(c["into"], acts)


@pytest.mark.parametrize("name", sorted(_G["seeded"]))
def test_golden_digest(ctx, name):
    seed, into = name[len("seed_"):].split("/")
    spec, steps = sc.seeded_steps(int(seed), moving=int(seed) % 3 != 0)
    assert rows_digest(_golden_device(ctx, spec, steps, into)) == _G["seeded"][name]["sha256"]


def test_merge_tree_in_rows(ctx):
    """The chain case's session holds two nested intervals, outer first (pre-order)."""
    spec, st, _ = CASES["chain_one_flush"]
    E = [r for call in run_device(ctx, spec, st.steps) for r in call[0]]
    assert len(E) == 1
    (s0, e0), (s1, e1) = E[0][3][1]
    assert s0 < s1 < e1 <= e0


def test_handles_any_u64(ctx):
    rnd = random.Random(5)
    spec, steps = sc.seeded_steps(4)
    vals = [0, 2**64 - 1] + [rnd.getrandbits(64) for _ in range(2000)]
    it = iter(vals)
    mapped = {}
    steps2 = []
    for s in steps:
        if s[0] == "batch":
            hs = []
            for v in s[4]:
                mapped[v] = next(it)
                hs.append(mapped[v])
            steps2.append(s[:4] + [hs])
        else:
            steps2.append(s)
    got = run_device(ctx, spec, steps2)
    want = run_device(ctx, spec, steps)
    inv = {v: k for k, v in mapped.items()}
    back = [([[r[0], r[1], r[2], [[inv[h] for h in r[3][0]], r[3][1]]] for r in E], M, [[r[0], r[1], r[2], inv[r[3]]] for r in L],
             sorted(inv[h] for h in rel)) for E, M, L, rel in got]
    assert back == want


def test_apply_device_matches_apply(ctx):
    for seed in (1, 8, 19, 30):
        spec, steps = sc.seeded_steps(seed)
        assert run_device(ctx, spec, steps, device_cols=True) == run_device(ctx, spec, steps)


def _big_stream(seed, n_act, rows, n_keys, moving=True, spread=4 * S):
    rnd = random.Random(seed)
    now, base, steps, nxt = A + 50 * S, A, [], 0
    for _ in range(n_act):
        if moving:
            now += rnd.randint(0, 2 * S)
            if rnd.random() < 0.2:
                steps.append(["notify", now])
        keys = [rnd.randrange(n_keys) for _ in range(rows)]
        ts = [base + rnd.randint(-spread, spread) - (rnd.randint(5 * S, 20 * S) if rnd.random() < 0.05 else 0) for _ in range(rows)]
        steps.append(["batch", now, keys, ts, list(range(nxt, nxt + rows))])
        nxt += rows
        base += S
    return steps


@pytest.mark.parametrize("ordered", [False, True])
def test_random_streams_1000_keys(ctx, ordered):
    spec = dict(ordered=ordered, gap_us=2 * S, wait_us=S)
    steps = _big_stream(3 + ordered, 25, 4000, 1000)
    n = _check(ctx, spec, steps)
    assert ordered or n > 0


def test_store_growth_keeps_retagged_entries(ctx):
    """Small batches into a store that starts at one batch: it grows and is compacted many times while merged-away
    sessions' entries are retagged; wait forever keeps most sessions open until EOF."""
    spec = dict(ordered=False, gap_us=3 * S, wait_us=20 * S)
    steps = _big_stream(9, 60, 300, 40, spread=8 * S)
    assert _check(ctx, spec, steps, max_batch_rows=300) > 0


def test_hot_key_one_long_session(ctx):
    n = 100_000
    rnd = random.Random(2)
    ts = [A + i * 1000 + rnd.randint(0, 5000) for i in range(n)]
    steps = [["batch", A, [7] * n, ts, list(range(n))]]
    _check(ctx, dict(ordered=False, gap_us=S, wait_us=F), steps, max_batch_rows=n)


def _expect(fn, status, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == status and what in str(ei.value), str(ei.value)


def _refused(j):
    with pytest.raises(N.BwError) as ei:
        j.advance()
    assert ei.value.status == 5


def test_sessions_per_key_exactly_full(ctx):
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, spec_(gap=0), max_sessions_per_key=4)
        try:
            n = 4 + extra
            call = lambda: j.apply(np.full(n, 3, np.uint64), np.arange(n), A + np.arange(n, dtype=np.int64) * S)  # noqa: E731
            if ok:
                call()
                out = j.eof()
                assert out.down_window_id.tolist() == [0, 1, 2, 3] and sorted(out.released.tolist()) == [0, 1, 2, 3]
            else:
                _expect(call, 3, "max_sessions_per_key")
                _refused(j)
        finally:
            j.close()


def test_merge_intervals_exactly_full(ctx):
    """M = 3.  A chain in one call gives session 0 two intervals but one merged id; two more merges give it four
    intervals (three merged ids), one past M."""
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, spec_(gap=10 * S), max_sessions_per_key=3)
        try:
            nxt = [0]

            def call(*ts):
                j.apply(np.full(len(ts), 3, np.uint64), np.arange(len(ts)) + nxt[0], np.array(ts, np.int64))
                nxt[0] += len(ts)

            call(A, A + 20 * S, A + 40 * S)
            call(A + 30 * S, A + 10 * S)  # 2 into 1, 1 into 0: intervals 2
            call(A + 60 * S)
            call(A + 50 * S)  # 3 into 0: intervals 3 == M
            if ok:
                out = j.eof()
                assert [len(out.merges(i)) for i in range(out.down_key.size)] == [3]
            else:
                call(A + 80 * S)
                _expect(lambda: call(A + 70 * S), 3, "merge intervals")
                _refused(j)
        finally:
            j.close()


def test_sessions_and_intervals_full_at_64(ctx):
    """M = 64, the engine's: 64 sessions of one key fill every cell; one call of bridges merges 63 of them into session 0
    (63 intervals); one more merge makes 64 intervals, exactly full; the next is one past."""
    spec = spec_(gap=10 * S)
    st = Steps().batch(*[(3, A + 20 * i * S) for i in range(64)]).batch(*[(3, A + (20 * i + 10) * S) for i in range(63)])
    st.batch((3, A + 64 * 20 * S)).batch((3, A + (63 * 20 + 10) * S))
    assert _check(ctx, spec, st.steps) == 64
    last = run_device(ctx, spec, st.steps)[-1]
    assert len(last[0]) == 1 and len(last[0][0][3][1]) == 64 and len(last[1][0][3][2]) == 64
    j = _mk(ctx, spec)
    try:
        n = 0
        for s in st.steps:
            j.apply(np.array(s[2], np.uint64), np.array(s[4], np.uint64), np.array(s[3], np.int64))
            n = s[4][-1] + 1
        j.apply(np.array([3], np.uint64), np.array([n]), np.array([A + 65 * 20 * S], np.int64))
        # (the 65th merge passes both the merged-id and the interval limit)
        _expect(lambda: j.apply(np.array([3], np.uint64), np.array([n + 1]), np.array([A + (64 * 20 + 10) * S], np.int64)), 3,
                "merge intervals")
        _refused(j)
    finally:
        j.close()
    for extra, ok in ((0, True), (1, False)):  # 64 sessions during a call, then 65
        j = _mk(ctx, spec_(gap=0))
        try:
            n = 64 + extra
            call = lambda: j.apply(np.full(n, 3, np.uint64), np.arange(n), A + np.arange(n, dtype=np.int64) * S)  # noqa: E731
            if ok:
                call()
                out = j.eof()
                assert out.down_window_id.tolist() == list(range(64)) and out.lists() == [[i] for i in range(64)]
            else:
                _expect(call, 3, "max_sessions_per_key")
                _refused(j)
        finally:
            j.close()


def test_queue_pool_exactly_full(ctx):
    j = _mk(ctx, spec_(ordered=True), max_queued_rows=10)
    try:
        j.apply(np.arange(6, dtype=np.uint64), np.arange(6), np.full(6, A, np.int64))
        j.apply(np.arange(4, dtype=np.uint64), np.arange(4) + 6, np.full(4, A + S, np.int64))
        assert j.advance().down_key.size == 0
        _expect(lambda: j.apply(np.array([9], np.uint64), np.array([10]), np.array([A], np.int64)), 3, "max_queued_rows")
        _refused(j)
    finally:
        j.close()
    j = _mk(ctx, spec_(ordered=True), max_queued_rows=10)
    try:
        j.apply(np.arange(10, dtype=np.uint64), np.arange(10), np.full(10, A, np.int64))
        out = j.eof()
        assert out.down_key.size == 10 and sorted(out.released.tolist()) == list(range(10))
    finally:
        j.close()


def test_late_and_emit_buffers_exactly_full(ctx):
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, spec_(gap=0, wait=0), max_late_rows=4)
        try:
            j.apply(np.array([1], np.uint64), np.array([0]), np.array([A + 100 * S], np.int64))
            n = 4 + extra
            call = lambda: j.apply(np.full(n, 1, np.uint64), np.arange(n) + 10, np.full(n, A, np.int64))  # noqa: E731
            if ok:
                call()
                assert j.advance().late_key.size == 4
            else:
                _expect(call, 3, "max_late_rows")
        finally:
            j.close()
    for extra, ok in ((0, True), (1, False)):
        j = _mk(ctx, spec_(gap=0, wait=0), max_emit_rows=4)
        try:
            n = 4 + extra
            call = lambda: j.apply(np.arange(n, dtype=np.uint64), np.arange(n), np.full(n, A, np.int64))  # noqa: E731
            call()
            if ok:
                assert j.eof().down_key.size == 4
            else:
                _expect(j.eof, 3, "max_emit_rows")
        finally:
            j.close()


def test_key_table_exactly_full(ctx):
    j = _mk(ctx, spec_(gap=S, wait=0), capacity_hint=16)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, 2**64 - 1], dtype=np.uint64)
        j.apply(keys, np.arange(keys.size), np.full(keys.size, A, np.int64))
        assert j.advance().down_key.size == 0
        _expect(lambda: j.apply(np.array([2000], np.uint64), np.array([1]), np.array([A], np.int64)), 3, "key table full")
        _refused(j)
    finally:
        j.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle():
        j = gpu.SessionCollectWindow(ctx, True, S, S, capacity_hint=1 << 16, max_sessions_per_key=16)
        rnd = random.Random(1)
        keys = np.array([rnd.randrange(5000) for _ in range(20000)], np.uint64)
        j.apply(keys, np.arange(keys.size), A + np.arange(keys.size, dtype=np.int64) * 1000)
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
