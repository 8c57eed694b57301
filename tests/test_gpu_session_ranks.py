"""K7, the session-window fold, sharded by key over W ranks: threads of one process on a loopback world (include/bwgpu.h,
bw_loopback_create), whose partition kernels, peer stores into the owners' receive regions and barriers are the ones an
NCCL world runs.  -m gpu.

Each rank applies its own rows per call; each row goes to rank `po.dest_rank(key, W)`, which folds what arrived in
(source rank, source order).  The rows of all ranks of one call, the closed and the late columns each stably sorted by
key string, must equal what a world-1 fold returns for the rank-major concatenation of every rank's columns: the
reference's rows (tests/golden/session_cases.json, `so.run_sessions`) and a world-1 `SessionFold`, f64 bits included.
A late row (rank r, row i) of an activation is world-1 row offset_r + i."""

import itertools
import json
import os
import random
import time

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po  # checker only
from oracle.streams import rows_digest
from tests import session_oracle as so
from tests.test_gpu_join_ranks import no_errors, run_ranks
from tests.test_gpu_sessions import _rows, _same

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
S, A = so.S, so.A
SENTINEL = 2**64 - 1  # the key table's empty marker; the key itself lives in the alias slot `cap`
WORLDS = [2, 3, 4]
BARRIER_TIMEOUT_S = 120  # the loopback world's barrier gives up after this long
SMALL = dict(capacity_hint=64, max_emit_rows=4096, max_late_rows=4096)  # the golden and seeded streams' tables

with open(os.path.join(os.path.dirname(__file__), "golden", "session_cases.json")) as _f:
    GOLDEN = json.load(_f)


def _fold(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    return gpu.SessionFold(ctx, spec["reduction"], spec["gap_us"], None if wait == so.WAIT_FOREVER else wait,
                           val_dtype=spec.get("val_dtype", "i64"), shard_by_key=True, **kw)


def _cols(spec, step, idx=None):
    _, _, keys, ts, vals = step
    dt = np.float64 if spec.get("val_dtype") == "f64" else np.int64
    k, t, v = np.array(keys, np.uint64), np.array(ts, np.int64), np.array(vals, dt)
    if idx is not None:
        k, t, v = k[idx], t[idx], v[idx]
    return k, None if spec["reduction"] == "count" else v, t


# ---- splits of one batch of n rows into per-rank index arrays --------------------------------------------------------


def contiguous(world, seed):
    """Contiguous slices (the rank-major concatenation is the batch itself), cycling per batch through even cuts, every
    row on one rank, and seeded cuts that leave some ranks empty."""
    rnd = random.Random(seed)

    def split(i, n):
        mode = (i + seed) % 3
        if mode == 0:
            cuts = [n * r // world for r in range(world + 1)]
        elif mode == 1:
            owner = i % world
            cuts = [0] * (owner + 1) + [n] * (world - owner)
        else:
            cuts = [0] + sorted(rnd.randint(0, n) for _ in range(world - 1)) + [n]
        return [np.arange(cuts[r], cuts[r + 1]) for r in range(world)]

    return split


def interleaved(world):
    return lambda i, n: [np.arange(r, n, world) for r in range(world)]


def random_split(world, seed):
    rnd = np.random.default_rng(seed)

    def split(i, n):
        to = rnd.integers(0, world, n)
        return [np.flatnonzero(to == r) for r in range(world)]

    return split


# ---- the drivers ------------------------------------------------------------------------------------------------------


def plan(steps, world, split):
    """Per step: the per-rank index arrays of a batch (None for notify) and the rank-major concatenation's steps."""
    parts, cat = [], []
    for i, step in enumerate(steps):
        if step[0] != "batch":
            parts.append(None)
            cat.append(step)
            continue
        p = split(i, len(step[2]))
        order = np.concatenate(p).astype(np.int64) if p else np.zeros(0, np.int64)
        assert sorted(order.tolist()) == list(range(len(step[2])))
        parts.append(p)
        cat.append(["batch", step[1]] + [[step[c][j] for j in order.tolist()] for c in (2, 3, 4)])
    return parts, cat


def run_world(world, spec, steps, parts, **kw):
    """Every rank plays every step with its slice, then EOF.  Per rank: its SessionRows per call."""

    def body(r, ctx, keep):
        f = _fold(ctx, spec, **kw)
        keep.append(f)
        out = []
        for i, step in enumerate(steps):
            if step[0] == "batch":
                f.apply(*_cols(spec, step, parts[i][r]), epoch=i + 1, system_now_us=step[1])
                out.append(f.advance())
            else:
                out.append(f.advance(system_now_us=step[1]))
        out.append(f.eof())
        return out

    results, errors = run_ranks(world, body)
    no_errors(errors)
    return results


def run_one(spec, steps, **kw):
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    f = _fold(ctx, spec, **kw)
    out = []
    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                f.apply(*_cols(spec, step), epoch=i + 1, system_now_us=step[1])
                out.append(f.advance())
            else:
                out.append(f.advance(system_now_us=step[1]))
        out.append(f.eof())
    finally:
        f.close()
        ctx.close()
    return out


def merge(outs, world, offsets):
    """Every rank's SessionRows of one call as one world-1 SessionRows: the closed and the late columns concatenated and
    each stably sorted by key string; late rows renamed to rows of the rank-major concatenation (offsets[r] rows come
    before rank r's).  Checks that each rank returned only keys it owns."""
    from bytewax_b200 import gpu

    for r, o in enumerate(outs):
        assert all(po.dest_rank(k, world) == r for k in np.unique(np.concatenate([o.closed_key, o.late_key])).tolist()), r
        assert (o.late_rank < world).all()  # the source rank, which need not be the owner

    def cat(name):
        return np.concatenate([getattr(o, name) for o in outs])

    ck, lk = cat("closed_key"), cat("late_key")
    co = np.argsort(ck.astype(str), kind="stable")
    lo = np.argsort(lk.astype(str), kind="stable")
    mids = [o.merged(i) for o in outs for i in range(o.closed_key.size)]
    mids = [mids[i] for i in co.tolist()]
    off = np.zeros(len(mids) + 1, np.int64)
    off[1:] = np.cumsum([len(m) for m in mids])
    ids = np.array(list(itertools.chain.from_iterable(mids)), np.int64)
    rank, row = cat("late_rank"), cat("late_row")
    base = np.array(offsets or [0] * world, np.uint64)[rank.astype(np.int64)]
    return gpu.SessionRows(ck[co], cat("closed_window_id")[co], cat("closed_acc")[co], cat("closed_open_us")[co],
                           cat("closed_close_us")[co], cat("closed_epoch")[co], off, ids, lk[lo], cat("late_epoch")[lo],
                           cat("late_activation")[lo], (base + row)[lo], np.zeros(lk.size, np.uint64))


def merged_calls(results, world, cat, parts):
    """Per call (each step of the rank-major concatenation `cat`, then EOF): the merged SessionRows and the
    reference-format rows."""
    steps = cat
    out, n_act = [], 0
    for i in range(len(steps) + 1):
        step = steps[i] if i < len(steps) else None
        if step is not None and step[0] == "batch":
            sizes = [len(p) for p in parts[i]]
            offsets = [sum(sizes[:r]) for r in range(world)]
            m = merge([results[r][i] for r in range(world)], world, offsets)
            out.append((m, _rows(m, (n_act, step[4]))))
            n_act += 1
        else:
            m = merge([results[r][i] for r in range(world)], world, None)
            assert m.late_key.size == 0
            out.append((m, _rows(m, None)))
    return out


COLS = ["closed_key", "closed_window_id", "closed_open_us", "closed_close_us", "closed_epoch", "merged_off", "merged_ids",
        "late_key", "late_epoch", "late_activation", "late_row"]


def same_rows(a, b):
    """Two SessionRows equal column for column, accumulators by their bits."""
    for c in COLS:
        assert np.array_equal(getattr(a, c), getattr(b, c)), c
    assert a.closed_acc.view(np.uint64).tolist() == b.closed_acc.view(np.uint64).tolist()


# ---- the reference's rows ---------------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_golden_case_ranks(name):
    case = GOLDEN["cases"][name]
    for world in WORLDS:
        for seed in range(3):  # each batch of the case meets each kind of contiguous split
            parts, cat = plan(case["steps"], world, contiguous(world, seed))
            assert cat == case["steps"]
            got = merged_calls(run_world(world, case["spec"], case["steps"], parts, max_batch_rows=64, **SMALL), world, case["steps"], parts)
            assert _same([rows for _, rows in got], case["acts"]), (world, seed)


@pytest.mark.parametrize("seed", list(so.SEEDED))
def test_seeded_digests_ranks(seed):
    spec, steps = so.seeded_steps(seed, moving=seed % 3 != 0)
    want = GOLDEN["seeded"][f"seed_{seed}"]
    for world in WORLDS:
        parts, _ = plan(steps, world, contiguous(world, seed))
        got = [rows for _, rows in merged_calls(run_world(world, spec, steps, parts, max_batch_rows=32, max_sessions_per_key=64, **SMALL),
                                                world, steps, parts)]
        assert [len(a) for a in got] == want["rows"], world
        assert rows_digest(got) == want["sha256"], world


def _stream(seed, n_act, rows, n_keys, fval=False, edge=True):
    rnd = np.random.default_rng(seed)
    steps, base, now = [], A, A + 100 * S
    for b in range(n_act):
        keys = rnd.integers(0, n_keys, rows).astype(np.uint64)
        if edge:
            keys[rnd.random(rows) < 0.002] = SENTINEL
            keys[rnd.random(rows) < 0.002] = 0
        ts = base + rnd.integers(-6 * S, 6 * S, rows) - np.where(rnd.random(rows) < 0.05, rnd.integers(5 * S, 40 * S, rows), 0)
        vals = rnd.choice(np.array(so.F64_VALUES), rows) if fval else rnd.integers(-1000, 1000, rows)
        now += int(rnd.integers(0, 2 * S))
        steps.append(["batch", now, keys.tolist(), ts.tolist(), vals.tolist()])
        if b % 2:
            steps.append(["notify", now + 3 * S])
        base += 3 * S
    return steps


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("how", ["interleaved", "random"])
@pytest.mark.parametrize("seed,red,dtype", [(1, "count", "i64"), (2, "sum", "f64"), (3, "max", "i64"), (4, "min", "f64")])
def test_splits_match_oracle_and_one_rank(world, how, seed, red, dtype):
    """Interleaved and seeded-random splits: merged rows == so.run_sessions == a world-1 SessionFold over the rank-major
    concatenation; late rows name the world-1 row; every key lands on one owner."""
    spec = dict(reduction=red, val_dtype=dtype, gap_us=1 * S, wait_us=2 * S)
    steps = _stream(seed, 5, 6000, 800, fval=dtype == "f64")
    split = interleaved(world) if how == "interleaved" else random_split(world, seed)
    parts, cat = plan(steps, world, split)
    kw = dict(capacity_hint=1 << 12, max_sessions_per_key=64)
    got = merged_calls(run_world(world, spec, steps, parts, max_batch_rows=6000, **kw), world, cat, parts)
    want = so.run_sessions(spec, cat)
    one = run_one(spec, cat, max_batch_rows=6000 * world, **kw)
    assert len(got) == len(want) == len(one)
    for i, ((m, rows), w, o) in enumerate(zip(got, want, one)):
        assert _same(rows, w), f"step {i}"
        same_rows(m, o)
    assert sum(m.late_key.size for m, _ in got) > 500 and sum(m.merged_ids.size for m, _ in got) > 200


def test_late_rows_name_their_source():
    """Late rows, one per rank, named (activation, rank, row in that rank's columns)."""
    world = 3
    spec = dict(reduction="sum", val_dtype="i64", gap_us=S, wait_us=0)
    keys = [1, 2, 3, 4, 5, 6]
    first = ["batch", A + 60 * S, keys, [A + 50 * S] * 6, [1] * 6]  # every key's watermark reaches A + 50 s
    # rank r holds rows [2r, 2r + 1] of the second batch: the second row of each rank is late
    second = ["batch", A + 61 * S, keys, [A + 51 * S, A, A + 52 * S, A + S, A + 53 * S, A + 2 * S], [10, 11, 12, 13, 14, 15]]
    steps = [first, second]
    parts, _ = plan(steps, world, lambda i, n: [np.arange(2 * r, 2 * r + 2) for r in range(world)])
    results = run_world(world, spec, steps, parts, max_batch_rows=8)
    late = sorted((k, int(a), int(rk), int(rw)) for o in (results[r][1] for r in range(world))
                  for k, a, rk, rw in zip(o.late_key.tolist(), o.late_activation, o.late_rank, o.late_row))
    assert late == [(2, 1, 0, 1), (4, 1, 1, 1), (6, 1, 2, 1)]
    one = run_one(spec, steps, max_batch_rows=8)[1]
    assert sorted(zip(one.late_key.tolist(), one.late_row.tolist())) == [(2, 1), (4, 3), (6, 5)]
    assert (one.late_rank == 0).all()


def test_edge_keys_on_different_owners():
    """Keys 0 and 2^64-1 (the alias slot) land on different ranks at W = 2, and every key of a stream on one owner."""
    world = 2
    assert po.dest_rank(0, world) != po.dest_rank(SENTINEL, world)
    spec = dict(reduction="sum", val_dtype="i64", gap_us=S, wait_us=S)
    steps = _stream(11, 4, 3000, 50)
    parts, cat = plan(steps, world, random_split(world, 11))
    results = run_world(world, spec, steps, parts, max_batch_rows=3000, capacity_hint=64)
    holders = {}
    for r in range(world):
        for o in results[r]:
            for k in o.closed_key.tolist() + o.late_key.tolist():
                holders.setdefault(k, set()).add(r)
    assert holders[0] == {po.dest_rank(0, world)} and holders[SENTINEL] == {po.dest_rank(SENTINEL, world)}
    assert all(len(h) == 1 for h in holders.values())
    got = merged_calls(results, world, cat, parts)
    assert all(_same(rows, w) for (_, rows), w in zip(got, so.run_sessions(spec, cat)))


@pytest.mark.parametrize("red,dtype", [("count", "i64"), ("sum", "i64"), ("sum", "f64"), ("max", "i64")])
def test_scale_four_ranks(red, dtype):
    """2^20 rows per rank over 10^5 keys at W = 4, against a world-1 fold of the concatenation, column for column."""
    world, rows, n_keys = 4, 1 << 20, 100_000
    spec = dict(reduction=red, val_dtype=dtype, gap_us=2 * S, wait_us=S)
    rnd = np.random.default_rng(20)
    dt = np.float64 if dtype == "f64" else np.int64
    acts = []
    for a in range(2):  # 10 s of event time each, 20 s apart: the first activation's sessions close in the second
        keys = rnd.integers(0, n_keys, rows * world).astype(np.uint64)
        ts = A + a * 20 * S + np.arange(rows * world, dtype=np.int64) * (10 * S) // (rows * world) + rnd.integers(-S, S + 1, rows * world)
        vals = rnd.choice(np.array(so.F64_VALUES), rows * world) if dtype == "f64" else rnd.integers(-10**6, 10**6, rows * world)
        acts.append((keys, None if red == "count" else vals.astype(dt), ts))
    kw = dict(capacity_hint=n_keys, max_emit_rows=1 << 19, max_late_rows=1 << 21, max_sessions_per_key=64)

    def body(r, ctx, keep):
        f = _fold(ctx, spec, max_batch_rows=rows, **kw)
        keep.append(f)
        out = []
        for a, (k, v, t) in enumerate(acts):
            sl = slice(r * rows, (r + 1) * rows)
            f.apply(k[sl], None if v is None else v[sl], t[sl], epoch=a + 1)
            out.append(f.advance())
        out.append(f.eof())
        return out

    results, errors = run_ranks(world, body)
    no_errors(errors)
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    f = _fold(ctx, spec, max_batch_rows=rows * world, **kw)
    one = []
    for a, (k, v, t) in enumerate(acts):
        f.apply(k, v, t, epoch=a + 1)
        one.append(f.advance())
    one.append(f.eof())
    f.close()
    ctx.close()
    closed = late = 0
    for i in range(len(acts) + 1):
        m = merge([results[r][i] for r in range(world)], world, [r * rows for r in range(world)] if i < len(acts) else None)
        same_rows(m, one[i])
        closed, late = closed + m.closed_key.size, late + m.late_key.size
    assert closed > n_keys and late > 1000


# ---- errors: every rank returns, none waits out a barrier -----------------------------------------------------------


def _errors_fast(world, body):
    t0 = time.monotonic()
    results, errors = run_ranks(world, body)
    assert time.monotonic() - t0 < BARRIER_TIMEOUT_S / 4, "a rank waited out a barrier"
    return results, errors


def _status(e):
    return e.status if isinstance(e, N.BwError) else e


@pytest.mark.parametrize("what", ["epoch", "now"])
def test_ranks_disagree(what):
    """Ranks that pass different epochs, or different system times, to one call: BW_ERR_STATE on every rank."""
    world = 3

    def body(r, ctx, keep):
        f = _fold(ctx, dict(reduction="count", gap_us=S, wait_us=0), capacity_hint=64, max_batch_rows=64)
        keep.append(f)
        f.apply(np.array([r, r + 1], np.uint64), None, np.array([A, A], np.int64), epoch=5, system_now_us=A)
        epoch, now = (6 if r == 2 else 7, A) if what == "epoch" else (6, A + (r == 1))
        f.apply(np.array([r], np.uint64), None, np.array([A], np.int64), epoch=epoch, system_now_us=now)
        return "no error"

    results, errors = _errors_fast(world, body)
    assert [_status(e) for e in errors] == [STATE] * world, (results, errors)


@pytest.mark.parametrize("what", ["rows", "null", "decreasing"])
def test_refused_call_folds_nothing(what):
    """One rank's call cannot go ahead (too many rows, a NULL column, a decreasing epoch): that rank gets its own error,
    every other rank BW_ERR_STATE, no rank folds the call, and the fold goes on as if it had not been made."""
    world, B = 3, 16
    spec = dict(reduction="sum", val_dtype="i64", gap_us=S, wait_us=S)
    steps = _stream(5, 3, 30, 20, edge=False)
    parts, cat = plan(steps, world, interleaved(world))
    bad = 1

    def body(r, ctx, keep):
        f = _fold(ctx, spec, max_batch_rows=B)
        keep.append(f)
        out, err = [], None
        for i, step in enumerate(steps):
            if i == 1:  # the refused call, between two good ones
                try:
                    if r == bad and what == "rows":
                        f.apply(np.zeros(B + 1, np.uint64), np.zeros(B + 1, np.int64), np.full(B + 1, A, np.int64), epoch=2, system_now_us=step[1])
                    elif r == bad and what == "null":
                        f.apply_device(0, 0, 0, 4, epoch=2, system_now_us=step[1])
                    else:
                        f.apply(*_cols(spec, step, parts[i][r]), epoch=0 if (r == bad and what == "decreasing") else 2,
                                system_now_us=step[1])
                except N.BwError as ex:
                    err = ex.status
                out.append(f.advance())
            if step[0] == "batch":
                f.apply(*_cols(spec, step, parts[i][r]), epoch=i + 1, system_now_us=step[1])
                out.append(f.advance())
            else:
                out.append(f.advance(system_now_us=step[1]))
        out.append(f.eof())
        return err, out

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    want_bad = SPEC if what in ("rows", "null") else STATE
    assert [e for e, _ in results] == [STATE if r != bad else want_bad for r in range(world)]
    assert all(o.closed_key.size == 0 and o.late_key.size == 0 for _, out in results for o in [out[1]])
    outs = [[o for j, o in enumerate(out) if j != 1] for _, out in results]
    got = merged_calls(outs, world, cat, parts)
    assert all(_same(rows, w) for (_, rows), w in zip(got, so.run_sessions(spec, cat)))


def _owned_by(rank, world, n, start=1):
    out, k = [], start
    while len(out) < n:
        if po.dest_rank(k, world) == rank:
            out.append(k)
        k += 1
    return out


@pytest.mark.parametrize("what", ["key table", "max_sessions_per_key"])
def test_owner_capacity(what):
    """An owner's key table (1024 slots at capacity_hint 16) or a key's session list fills up: that rank's apply gets
    BW_ERR_CAPACITY, every other rank goes on; every rank's next apply gets BW_ERR_STATE."""
    world, owner = 2, 0
    if what == "key table":
        keys = _owned_by(owner, world, 1025, start=10)  # one more than the table holds (key 2^64-1 has its own slot)
        ts = [A] * len(keys)
        kw = dict(capacity_hint=16)
    else:
        keys = _owned_by(owner, world, 1) * 5  # five sessions, 10 s apart, for one key that may hold four
        ts = [A + i * 10 * S for i in range(5)]
        kw = dict(max_sessions_per_key=4)
    parts = [np.arange(r, len(keys), world) for r in range(world)]

    def body(r, ctx, keep):
        f = _fold(ctx, dict(reduction="count", gap_us=S, wait_us=None if what != "key table" else 0), max_batch_rows=1024, **kw)
        keep.append(f)
        st = []
        for epoch in (1, 2):
            try:
                idx = parts[r] if epoch == 1 else []
                f.apply(np.array(keys, np.uint64)[idx], None, np.array(ts, np.int64)[idx], epoch=epoch)
                st.append(0)
            except N.BwError as ex:
                st.append(ex.status)
        return st

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    assert results[owner] == [CAPACITY, STATE] and results[1 - owner] == [0, STATE], results


def test_sharding_is_opt_in():
    """Without shard_by_key every rank of a world of 2 gets BW_ERR_SPEC at create, at once (no collective is entered);
    with it every rank creates the fold.  On one rank the flag changes nothing."""
    from bytewax_b200 import gpu

    def body(r, ctx, keep):
        with pytest.raises(N.BwError) as ei:
            gpu.SessionFold(ctx, max_batch_rows=1024, **SMALL)
        assert ei.value.status == SPEC and "one GPU" in str(ei.value)
        keep.append(gpu.SessionFold(ctx, max_batch_rows=1024, shard_by_key=True, **SMALL))
        return r

    results, errors = _errors_fast(2, body)
    no_errors(errors)
    assert results == [0, 1]
    steps = so.seeded_steps(7)[1]
    spec = so.seeded_spec(7)
    flagged, plain = run_one(spec, steps, max_sessions_per_key=64), _fold_plain_world1(spec, steps)
    assert len(flagged) == len(plain) == len(steps) + 1
    for a, b in zip(flagged, plain):
        same_rows(a, b)


def _fold_plain_world1(spec, steps):
    """A world-1 fold created without shard_by_key, driven like run_one."""
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    wait = spec["wait_us"]
    f = gpu.SessionFold(ctx, spec["reduction"], spec["gap_us"], None if wait == so.WAIT_FOREVER else wait,
                        val_dtype=spec.get("val_dtype", "i64"), max_sessions_per_key=64)
    out = []
    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                f.apply(*_cols(spec, step), epoch=i + 1, system_now_us=step[1])
                out.append(f.advance())
            else:
                out.append(f.advance(system_now_us=step[1]))
        out.append(f.eof())
    finally:
        f.close()
        ctx.close()
    return out


def test_spec_without_shard_field():
    """A spec whose struct_size ends before shard_by_key (built against the header without it) still creates a world-1
    fold; one of any other size is BW_ERR_SPEC."""
    import ctypes as C

    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    try:
        for size, ok in ((N.BwSessionSpec.shard_by_key.offset, True), (C.sizeof(N.BwSessionSpec) - 4, False)):
            s = N.BwSessionSpec()
            s.struct_size = size
            s.reduction, s.val_dtype, s.max_sessions_per_key = N.RED["count"], N.VAL["i64"], 4
            s.gap_us, s.capacity_hint, s.max_batch_rows, s.max_emit_rows, s.max_late_rows = S, 64, 64, 64, 64
            s.shard_by_key = 1
            h = C.c_void_p()
            st = ctx.lib.bw_session_create(ctx.h, C.byref(s), C.byref(h))
            assert (st == 0) == ok, size
            if st == 0:
                ctx.lib.bw_session_destroy(h)
    finally:
        ctx.close()


@pytest.mark.parametrize("world,rows", [(2, 1 << 30), (3, 715_827_883), (4, 1 << 29), (8, 1 << 28)])
def test_batch_limit(world, rows):
    """max_batch_rows x world reaching 2^31 is BW_ERR_SPEC at create, on every rank."""
    assert rows * world >= 2**31 and (rows - 1) * world < 2**31

    def body(r, ctx, keep):
        keep.append(_fold(ctx, dict(reduction="count", gap_us=S, wait_us=0), max_batch_rows=rows))

    _, errors = _errors_fast(world, body)
    assert [_status(e) for e in errors] == [SPEC] * world, errors


def test_memory_returned_on_destroy():
    """Create, use and destroy a W = 2 fold three times: device memory comes back (regions, mappings, scratch)."""
    spec = dict(reduction="sum", val_dtype="f64", gap_us=S, wait_us=S)
    steps = _stream(3, 3, 2000, 300, fval=True)
    parts, _ = plan(steps, 2, interleaved(2))

    def cycle():
        run_world(2, spec, steps, parts, capacity_hint=1 << 14, max_batch_rows=1 << 16, max_sessions_per_key=32)

    cycle()  # warm the allocator's pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        cycle()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
