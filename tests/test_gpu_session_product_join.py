"""K16: `join_window(insert_mode="product")` over session windows on the device (`bw_spjwin_*`) against the reference's
own session product joins.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/session_product_join_cases.json
(made by the reference's `_WindowLogic` + `_SessionWindowerLogic` + `_JoinWindowLogic`,
tools/gen_session_product_join_golden.py), the SHA-256 digests of its seeded streams, and
`tests/session_product_join_oracle.run_session_product_join` on larger streams -- including the handles each call
releases."""

import json
import os

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import session_product_join_oracle as sp

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = sp.S, sp.A
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE


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
    return gpu.SessionProductJoinWindow(ctx, spec["emit_mode"], spec["ordered"], spec["sides"], spec["gap_us"],
                                        None if wait == sp.WAIT_FOREVER else wait, **kw)


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
    late rows (arrival order), its down rows, its meta rows (id order).  Under `final` every down row is a close's: each
    closing session's product (at least one row) comes as one run of its id, in the order of the meta rows, and each run
    goes before its meta row; otherwise every down row goes before the key's meta rows."""
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
        if not final:
            rows.extend([k, dw[i], "E", list(dt[i])] for i in di)
        at = 0
        for i in mi:
            if final:
                assert at < len(di) and dw[di[at]] == mw[i], "a closing session without its final rows"
                while at < len(di) and dw[di[at]] == mw[i]:
                    rows.append([k, mw[i], "E", list(dt[di[at]])])
                    at += 1
            rows.append([k, mw[i], "M", [mo[i], mc[i], out.merged(i)]])
        assert not final or at == len(di), "final rows of a session that did not close"
    return rows


def run_device(ctx, spec, steps, device_cols=False, **kw):
    """Drive a SessionProductJoinWindow through golden-format steps: (rows, sorted released handles) per step, then EOF."""
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
                    torch.cuda.synchronize()
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


def _released_once(steps, released):
    flat = [h for r in released for h in r]
    assert len(flat) == len(set(flat)), "a handle released twice"
    assert set(flat) == {v for st in steps if st[0] == "batch" for v in st[5]}, "a handle never released"


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "session_product_join_cases.json")


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
    assert released == sp.run_session_product_join(case["spec"], case["steps"])[1]
    _released_once(case["steps"], released)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case_other_order(ctx, golden, name):
    """The same steps with `ordered` flipped, against the oracle (which matches every golden case)."""
    case = golden["cases"][name]
    spec = dict(case["spec"], ordered=not case["spec"]["ordered"])
    assert run_device(ctx, spec, case["steps"]) == sp.run_session_product_join(spec, case["steps"])


@pytest.mark.parametrize("seed", list(sp.SEEDED))
def test_seeded_digests(ctx, golden, seed):
    g = golden["seeded"][f"seed_{seed}"]
    spec, steps = sp.seeded_steps(seed, moving=seed % 3 != 0)
    acts, released = run_device(ctx, spec, steps)
    assert [len(a) for a in acts] == g["rows"]
    assert rows_digest(acts) == g["sha256"]
    assert released == sp.run_session_product_join(spec, steps)[1]


def _stream(seed, spec, n_keys, n_steps, per_step, moving=True):
    """Activations over n_keys keys: timestamps within +-3 s of a base that moves 1 s per activation, one item in twenty
    up to 30 s behind; with `moving`, the system clock steps and every third activation is followed by a notify."""
    rnd = np.random.default_rng(seed)
    steps, nxt, now, base = [], 0, A + 50 * S, A
    for i in range(n_steps):
        if moving:
            now += int(rnd.integers(0, 3 * S))
        keys = rnd.integers(0, n_keys, per_step).tolist()
        late = np.where(rnd.random(per_step) < 0.05, rnd.integers(5 * S, 30 * S, per_step), 0)
        ts = (base + rnd.integers(-3 * S, 3 * S, per_step) - late).tolist()
        sides = rnd.integers(0, spec["sides"], per_step).tolist()
        steps.append(["batch", now, keys, ts, sides, list(range(nxt, nxt + per_step))])
        nxt += per_step
        base += S
        if moving and i % 3 == 2:  # (the system clock never goes backwards)
            now += S
            steps.append(["notify", now])
    return steps


@pytest.mark.parametrize("emit", list(sp.EMITS))
@pytest.mark.parametrize("ordered", [True, False])
def test_streams_match_oracle(ctx, emit, ordered):
    i = sp.EMITS.index(emit)
    n_keys = (1000, 10_000, 100_000)[i]
    spec = dict(emit_mode=emit, ordered=ordered, sides=1 + (i + 2 * ordered) % 4, gap_us=S, wait_us=2 * S)
    steps = _stream(300 + i * 2 + ordered, spec, n_keys, 8, max(n_keys // 4, 3000))
    stats = {}
    want = sp.run_session_product_join(spec, steps, stats=stats)
    got = run_device(ctx, spec, steps, capacity_hint=n_keys)
    assert got[0] == want[0]
    assert got[1] == want[1]
    _released_once(steps, got[1])
    assert sum(len(a) for a in want[0]) > 1000
    assert (stats["merges"] > 0) == (not ordered)  # ordered streams never merge


def test_chain_of_62_merges_in_one_call(ctx):
    """One key holds 63 live sessions (3 s apart, gap 2 s) at max_sessions_per_key=64; then one batch bridges every
    adjacent pair from the top down, so the merge queue chains (62 -> 61, 61 -> 60, ..., 1 -> 0): under `running`, 62
    insert emissions, then 62 merge emissions in queue order, each in exact product order."""
    spec = dict(emit_mode="running", ordered=False, sides=2, gap_us=2 * S, wait_us=sp.WAIT_FOREVER)
    t = [A + 3 * S * i for i in range(63)]
    first = ["batch", A, [9] * 63, t, [i % 2 for i in range(63)], list(range(63))]
    bridge = ["batch", A, [9] * 62, [t[i] + 3 * S // 2 for i in range(61, -1, -1)], [(i + 1) % 2 for i in range(61, -1, -1)],
              list(range(63, 125))]
    steps = [first, bridge]
    stats = {}
    want = sp.run_session_product_join(spec, steps, stats=stats)
    assert stats["merges"] == 62
    got = run_device(ctx, spec, steps, max_sessions_per_key=64)
    assert got == want
    assert len({tuple(r[3]) for r in want[0][1] if r[1] == 0}) > 1000


def test_hot_key_one_long_session(ctx):
    """One key, 10^5 values in one session (1 us apart, gap 1 s): its `final` product, 3 x (10^5 - 3) rows, in order."""
    n = 100_000
    spec = dict(emit_mode="final", ordered=False, sides=2, gap_us=S, wait_us=sp.WAIT_FOREVER)
    j = _join(ctx, spec, max_batch_rows=n)
    try:
        rnd = np.random.default_rng(7)
        sides = np.zeros(n, np.uint8)
        sides[rnd.choice(n, 3, replace=False)] = 1
        vals = rnd.permutation(np.arange(n, dtype=np.uint64) + np.uint64(2**63))
        j.apply(np.full(n, 5, np.uint64), sides, vals, A + np.arange(n, dtype=np.int64))
        assert j.advance().down_key.size == 0
        out = j.eof()
        l0, l1 = vals[sides == 0], vals[sides == 1]
        assert out.down_key.size == l0.size * 3
        assert np.array_equal(out.down_handles[:, 0], np.repeat(l0, 3))
        assert np.array_equal(out.down_handles[:, 1], np.tile(l1, l0.size))
        assert (out.down_window_id == 0).all() and out.meta_key.tolist() == [5]
        assert out.meta_open_us.tolist() == [A] and out.meta_close_us.tolist() == [A + n - 1]
        assert sorted(out.released.tolist()) == sorted(vals.tolist())
    finally:
        j.close()


def test_max_product_rows_exactly_and_one_past(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=2, gap_us=10 * S, wait_us=S)
    keys, sides = np.full(7, 1, np.uint64), np.array([0, 0, 0, 1, 1, 1, 1], np.uint8)
    for limit, ok in ((12, True), (11, False)):
        j = _join(ctx, spec, max_product_rows=limit)
        try:
            j.apply(keys, sides, np.arange(7, dtype=np.uint64), np.full(7, A, np.int64))
            if ok:
                assert j.eof().down_key.size == 12
                continue
            with pytest.raises(N.BwError) as e:
                j.eof()
            assert e.value.status == CAPACITY and "max_product_rows" in str(e.value)
            with pytest.raises(N.BwError) as e:
                j.apply(keys, sides, np.arange(7, 14, dtype=np.uint64), np.full(7, A, np.int64))
            assert e.value.status == STATE
        finally:
            j.close()


def test_emit_buffer_exactly_full_and_one_past(ctx):
    spec = dict(emit_mode="running", ordered=False, sides=2, gap_us=S, wait_us=sp.WAIT_FOREVER)
    for n, ok in ((16, True), (17, False)):
        j = _join(ctx, spec, max_emit_rows=16)
        try:
            def run():
                j.apply(np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8), np.arange(n, dtype=np.uint64), np.full(n, A, np.int64))
                return j.advance()

            if ok:
                assert run().down_key.size == 16
            else:
                with pytest.raises(N.BwError) as e:
                    run()
                assert e.value.status == CAPACITY and "max_emit_rows" in str(e.value)
        finally:
            j.close()


def test_key_table_exactly_full_and_one_past(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=1, gap_us=S, wait_us=sp.WAIT_FOREVER)
    j = _join(ctx, spec, capacity_hint=1)  # 1024 slots + the alias slot
    try:
        j.apply(np.arange(1024, dtype=np.uint64), np.zeros(1024, np.uint8), np.arange(1024, dtype=np.uint64), np.full(1024, A, np.int64))
        assert j.advance().down_key.size == 0
        with pytest.raises(N.BwError) as e:
            j.apply(np.array([5000], np.uint64), np.zeros(1, np.uint8), np.array([9999], np.uint64), np.array([A], np.int64))
            j.advance()
        assert e.value.status == CAPACITY and "key table full" in str(e.value)
    finally:
        j.close()


def test_sessions_exactly_full_and_one_past(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=2, gap_us=S, wait_us=sp.WAIT_FOREVER)
    for n, ok in ((4, True), (5, False)):
        j = _join(ctx, spec, max_sessions_per_key=4)
        try:
            def run():
                j.apply(np.zeros(n, np.uint64), np.zeros(n, np.uint8), np.arange(n, dtype=np.uint64), A + 3 * S * np.arange(n, dtype=np.int64))
                return j.eof()

            if ok:
                assert run().meta_key.size == 4
            else:
                with pytest.raises(N.BwError) as e:
                    run()
                assert e.value.status == CAPACITY and "max_sessions_per_key" in str(e.value)
        finally:
            j.close()


def test_store_compaction_during_live_running_session(ctx):
    """Short sessions of many keys close and their entries are compacted away, many times over, while key 1 keeps one
    running session open and growing: every one of its emissions must still name the right handles."""
    import random

    spec = dict(emit_mode="running", ordered=False, sides=2, gap_us=S, wait_us=S)
    rnd = random.Random(3)
    steps, nxt = [], 0
    for i in range(40):
        k = [1] + [2 + rnd.randrange(50) for _ in range(30)]
        ts = [A + 5000 * S + i + 1] + [A + (1000 + i * 3 + rnd.randrange(3)) * S for _ in range(30)]
        sd = [rnd.randrange(2) for _ in range(31)]
        steps.append(["batch", A, k, ts, sd, list(range(nxt, nxt + 31))])
        nxt += 31
    want = sp.run_session_product_join(spec, steps)
    got = run_device(ctx, spec, steps, max_batch_rows=64)
    assert got == want
    assert sum(r[0] == 1 and r[2] == "E" for a in want[0] for r in a) > 300


def test_apply_device_matches_apply(ctx):
    spec = dict(emit_mode="complete", ordered=False, sides=3, gap_us=S, wait_us=S)
    steps = _stream(77, spec, 300, 10, 500, moving=False)
    assert run_device(ctx, spec, steps, device_cols=True) == run_device(ctx, spec, steps)
    spec = dict(spec, ordered=True, emit_mode="running")
    assert run_device(ctx, spec, steps, device_cols=True) == run_device(ctx, spec, steps)


def test_bad_device_side_is_a_spec_error(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=2, gap_us=S, wait_us=0)
    j = _join(ctx, spec)
    try:
        keys = torch.zeros(2, dtype=torch.int64, device="cuda")
        sides = torch.tensor([0, 2], dtype=torch.uint8, device="cuda")
        ts = torch.full((2,), A, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        j.apply_device(keys.data_ptr(), sides.data_ptr(), keys.data_ptr(), ts.data_ptr(), 2)
        with pytest.raises(N.BwError) as e:
            j.advance()
        assert e.value.status == SPEC
    finally:
        j.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    base = dict(emit_mode="final", ordered=True, sides=2, gap_us=S, wait_us=0)
    for bad in (dict(sides=0), dict(sides=5), dict(emit_mode="bogus"), dict(gap_us=-1), dict(wait_us=-1)):
        with pytest.raises(N.BwError) as e:
            _join(ctx, dict(base, **bad))
        assert e.value.status == SPEC, bad
    for kw in (dict(max_sessions_per_key=0), dict(max_sessions_per_key=65), dict(max_emit_rows=1 << 31), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as e:
            _join(ctx, base, **kw)
        assert e.value.status == SPEC, kw
    j = _join(ctx, base)
    try:  # a host side column is checked before anything runs
        with pytest.raises(N.BwError) as e:
            j.apply(np.array([1], np.uint64), np.array([2], np.uint8), np.array([1], np.uint64), np.array([A], np.int64))
        assert e.value.status == SPEC
    finally:
        j.close()
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as e:
            gpu.SessionProductJoinWindow(ctxs[0])
        assert e.value.status == SPEC and "one GPU" in str(e.value)
    finally:
        for c in ctxs:
            c.close()
    with pytest.raises(N.BwError):  # bw_sjwin keeps refusing product
        gpu.SessionJoinWindow(ctx, insert_mode="product")


def test_memory_returned_on_destroy(ctx):
    spec = dict(emit_mode="running", ordered=True, sides=2, gap_us=S, wait_us=S)
    steps = _stream(9, spec, 2000, 6, 4000, moving=False)
    run_device(ctx, spec, steps)  # warm the allocator's pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        run_device(ctx, spec, steps)
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
