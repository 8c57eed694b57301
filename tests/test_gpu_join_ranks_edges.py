"""K6, the two-sided keyed join, sharded by key over W ranks on loopback worlds (tests/test_gpu_join_ranks.py): the
reference's rows under every kind of split, every refusal on every rank, calls that fail on every rank followed by good
ones, a full owner on every rank, and the edge keys and batch sizes at every world size.  -m gpu.

A call that cannot go ahead on one rank still passes both barriers of the exchange, so every test that expects an
error also checks that every rank returned well before the loopback barrier would give up."""

import json
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po  # checker only
from tests.test_gpu_join_ranks import MODES, arrays, check_against_one_rank, concat, merged, no_errors, one_rank, run_ranks
from tests.test_gpu_join_window_ranks import SPLITS, _split
from tests.test_gpu_session_ranks import _errors_fast, _owned_by

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
SENTINEL = 2**64 - 1
WORLDS = [2, 3, 4]

with open(os.path.join(os.path.dirname(__file__), "golden", "keyed_cases.json")) as _f:
    GOLDEN = json.load(_f)["join"]


def _slices(split, i, keys, sides, vals):
    """One activation's columns dealt to the ranks by `split` (each rank's share keeps the items' order)."""
    return [([keys[j] for j in p.tolist()], [sides[j] for j in p.tolist()], [vals[j] for j in p.tolist()]) for p in split(i, len(keys))]


def _key_order(rows):
    return sorted(rows, key=lambda rw: (rw[1], po.key_str(rw[0][0])))


# ---- the reference's rows ---------------------------------------------------------------------------------------------


@pytest.mark.parametrize("how", SPLITS)
@pytest.mark.parametrize("case", range(len(GOLDEN)))
def test_golden_case_ranks(case, how):
    """Each golden case at W = 2, 3 and 4 under one kind of split.  One item per call, as the golden plays it: every
    rank's rows, merged and stably sorted by (epoch, key string), are the golden rows, each on its key's owner and
    carrying its item's epoch.  Then in activations of 25 items: the merged rows of every call are `po.run_join`'s and a
    world-1 join's over the rank-major concatenation."""
    from bytewax_b200 import gpu

    c = GOLDEN[case]
    im, em, items = c["insert_mode"], c["emit_mode"], c["items"]
    want = po.run_join([([k], [s], [v]) for k, s, v in items], im, em)
    assert [list(r) for a in want for r in a] == c["rows"]
    kw = dict(capacity_hint=64, max_batch_rows=32, max_emit_rows=1024)
    for world in WORLDS:
        split = _split(how, world, case)
        acts = [_slices(split, i, [k], [s], [v]) for i, (k, s, v) in enumerate(items)]

        def body(r, ctx, keep):
            j = gpu.KeyedJoin(ctx, im, em, **kw)
            keep.append(j)
            for i, per_rank in enumerate(acts):
                j.apply(*arrays(*per_rank[r]), epoch=i + 1)
            # one advance for every call: the rows come out by (epoch, key string, item order)
            return [list(zip(rows, ep.tolist())) for rows, ep in (j.advance(), j.eof())]

        results, errors = run_ranks(world, body)
        no_errors(errors)
        for r in range(world):
            for part in results[r]:
                assert all(po.dest_rank(row[0], world) == r for row, _ in part), (world, how, r)
        got = _key_order(sum((results[r][0] for r in range(world)), []))
        per_act = [[] for _ in items]
        for row, e in got:
            assert row[0] == items[e - 1][0], (world, how, e)  # the row of the item played with epoch e
            per_act[e - 1].append(row)
        eof = _key_order(sum((results[r][1] for r in range(world)), []))
        assert all(e == len(items) for _, e in eof)
        assert per_act + [[row for row, _ in eof]] == want, (world, how)

        acts25 = [_slices(split, a, *(list(col) for col in zip(*items[lo:lo + 25]))) for a, lo in enumerate(range(0, len(items), 25))]
        check_against_one_rank(world, acts25, im, em, [2 * a + 1 for a in range(len(acts25))], **kw)


# ---- errors: every rank returns, none waits out a barrier -----------------------------------------------------------


def _stream(seed, world, n_act, n=30, n_keys=20):
    """n_act activations of n items over n_keys keys, dealt round-robin to the ranks."""
    rnd = random.Random(seed)
    acts = []
    for _ in range(n_act):
        ks = [rnd.randrange(n_keys) for _ in range(n)]
        cols = (ks, [rnd.randrange(2) for _ in ks], [rnd.randrange(2**64 - 10**6) for _ in ks])
        acts.append([tuple(list(c[r::world]) for c in cols) for r in range(world)])
    return acts


def _junk(per_rank):
    """The same rows with other payloads: played by mistake, they would show in the rows that follow."""
    return [(k, s, [v + 10**6 for v in vals]) for k, s, vals in per_rank]


def _check_rows(results, world, acts, epochs, im, em, **kw):
    """Per rank, the (rows, epochs) of each advance and of eof: merged, they are `po.run_join`'s and a world-1 join's
    over the rank-major concatenation of `acts`; each rank's rows are its own keys', with the call's epoch."""
    want = po.run_join([concat(per_rank) for per_rank in acts], im, em)
    w1 = one_rank(acts, im, em, epochs, **dict(kw, max_batch_rows=kw["max_batch_rows"] * world))
    for i in range(len(acts) + 1):
        assert merged([results[r][i][0] for r in range(world)]) == want[i] == w1[i], i
    for r in range(world):
        for i, (rows, eps) in enumerate(results[r]):
            assert all(po.dest_rank(k, world) == r for k, _, _ in rows), (r, i)
            assert eps == [epochs[min(i, len(epochs) - 1)]] * len(rows), (r, i)
    assert sum(len(a) for a in want) > 20


REFUSALS = [(what, 3, bad) for what in ("rows", "null", "decreasing") for bad in range(3)]
REFUSALS += [("rows", world, bad) for world in (2, 4) for bad in range(world)]


@pytest.mark.parametrize("what,world,bad", REFUSALS)
def test_refused_call_plays_nothing(what, world, bad):
    """Rank `bad`'s call cannot go ahead (too many rows, a NULL column, an epoch below the last one): that rank gets its
    own error, every other rank BW_ERR_STATE, no rank plays the call (every advance after it is empty), and the join
    goes on as if it had not been made.  The call before it plays no rows at epoch 2, so that epoch 0 decreases."""
    B = 16
    im, em = "last", "running"  # every item played emits a row
    acts = _stream(f"refused-{what}-{world}-{bad}", world, 3)
    empty = [([], [], [])] * world
    played = [acts[0], empty, acts[1], acts[2]]
    epochs = [1, 2, 3, 4]

    def body(r, ctx, keep):
        from bytewax_b200 import gpu

        j = gpu.KeyedJoin(ctx, im, em, capacity_hint=64, max_batch_rows=B, max_emit_rows=1024)
        keep.append(j)
        out, err = [], None
        for i, per_rank in enumerate(played):
            j.apply(*arrays(*per_rank[r]), epoch=epochs[i])
            if i == 1:  # the refused call, between two good ones
                try:
                    if r == bad and what == "rows":
                        j.apply(np.zeros(B + 1, np.uint64), np.zeros(B + 1, np.uint8), np.arange(B + 1, dtype=np.uint64), epoch=2)
                    elif r == bad and what == "null":
                        err = j.lib.bw_join_apply(j.h, None, None, None, 4, 2)
                    else:
                        j.apply(*arrays(*_junk(acts[1])[r]), epoch=0 if (r == bad and what == "decreasing") else 2)
                except N.BwError as ex:
                    err = ex.status
            rows, ep = j.advance()
            out.append((rows, ep.tolist()))
        rows, ep = j.eof()
        return err, out + [(rows, ep.tolist())]

    # checked once every rank is done: a rank that stopped early would leave its peers waiting in the next call
    results, errors = _errors_fast(world, body)
    no_errors(errors)
    want_bad = STATE if what == "decreasing" else SPEC
    assert [e for e, _ in results] == [want_bad if r == bad else STATE for r in range(world)], results
    assert all(out[1] == ([], []) for _, out in results), [out[1] for _, out in results]
    _check_rows([out for _, out in results], world, played, epochs, im, em, max_batch_rows=B, capacity_hint=64, max_emit_rows=1024)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("what", ["epochs differ", "decreasing"])
def test_join_goes_on_after_failed_call(what, world):
    """A call that fails on every rank -- its ranks pass different epochs, or all pass the same epoch below the last --
    passes both barriers on every rank and changes no rank's state: every rank gets BW_ERR_STATE, and the three calls
    that follow at once give the rows of the stream without it."""
    im, em = "first", "running"
    acts = _stream(f"go-on-{what}-{world}", world, 5)
    played = [acts[0]] + acts[2:]
    epochs = [5, 8, 9, 10]

    def body(r, ctx, keep):
        from bytewax_b200 import gpu

        j = gpu.KeyedJoin(ctx, im, em, capacity_hint=64, max_batch_rows=16, max_emit_rows=1024)
        keep.append(j)
        j.apply(*arrays(*acts[0][r]), epoch=5)
        err = None
        try:  # before the advance, so that epoch 3 is below the last one
            j.apply(*arrays(*_junk(acts[1])[r]), epoch=(6 if r == world - 1 else 7) if what == "epochs differ" else 3)
        except N.BwError as ex:
            err = ex.status
        out = []
        for i, per_rank in enumerate(played):
            if i:
                j.apply(*arrays(*per_rank[r]), epoch=epochs[i])
            rows, ep = j.advance()
            out.append((rows, ep.tolist()))
        rows, ep = j.eof()
        return err, out + [(rows, ep.tolist())]

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    assert [e for e, _ in results] == [STATE] * world, results
    _check_rows([out for _, out in results], world, played, epochs, im, em, max_batch_rows=16, capacity_hint=64, max_emit_rows=1024)


def _overfill(what, owner, world):
    """The keys that overfill `what` on rank `owner` in one call, and the join's arguments."""
    if what == "key table":  # 1024 slots at capacity_hint 16, and one key more; 2^64-1 has a slot of its own
        keys = _owned_by(owner, world, 1025, start=10)
        if po.dest_rank(SENTINEL, world) == owner:
            keys.append(SENTINEL)
        return keys, dict(capacity_hint=16, max_emit_rows=4096)
    return _owned_by(owner, world, 11, start=10), dict(capacity_hint=64, max_emit_rows=10)  # 11 running rows, 10 fit


OWNERS = [(world, owner) for world in WORLDS for owner in range(world)]


@pytest.mark.parametrize("world,owner", OWNERS)
@pytest.mark.parametrize("what", ["key table", "emit buffer"])
def test_owner_capacity(what, world, owner):
    """Rank `owner`'s key table or emit buffer overflows in the first of three calls that also carry every rank's keys:
    every apply completes on every rank; only the owner's advances raise, exactly as a world-1 join fed the owner's
    rows does; every other rank's rows in every call are `po.run_join`'s for the keys it owns."""
    from bytewax_b200 import gpu

    im, em = "last", "running"
    over, kw = _overfill(what, owner, world)
    kw["max_batch_rows"] = 1024
    rnd = random.Random(f"capacity-{what}-{world}-{owner}")
    pool = [k for r in range(world) for k in _owned_by(r, world, 3, start=10**6)]  # 3 keys of every rank
    cat = []
    for c in range(3):
        ks = pool + (over if c == 0 else [])
        rnd.shuffle(ks)
        cat.append((ks, [rnd.randrange(2) for _ in ks], [rnd.randrange(2**64) for _ in ks]))
    acts = [[tuple(list(col[r::world]) for col in cols) for r in range(world)] for cols in cat]
    order = [np.concatenate([np.arange(r, len(cols[0]), world) for r in range(world)]).tolist() for cols in cat]
    cat = [tuple([col[i] for i in o] for col in cols) for cols, o in zip(cat, order)]  # rank-major

    def play(j, per_call):
        """Per call its advance's (rows, epochs) or status, then eof's; a failed apply is recorded, not raised, so that
        every rank makes every call."""
        got = []
        for c, cols in enumerate(per_call):
            try:
                j.apply(*arrays(*cols), epoch=c + 1)
            except N.BwError as ex:
                got.append(("apply", ex.status))
            try:
                rows, ep = j.advance()
                got.append((rows, ep.tolist()))
            except N.BwError as ex:
                got.append(ex.status)
        try:
            rows, ep = j.eof()
            got.append((rows, ep.tolist()))
        except N.BwError as ex:
            got.append(ex.status)
        return got

    def body(r, ctx, keep):
        j = gpu.KeyedJoin(ctx, im, em, **kw)
        keep.append(j)
        return play(j, [a[r] for a in acts])

    results, errors = _errors_fast(world, body)
    no_errors(errors)

    ctx = gpu.Context(0)
    try:
        j = gpu.KeyedJoin(ctx, im, em, **dict(kw, max_batch_rows=world * 1024))
        mine = [tuple([col[i] for i in range(len(ks)) if po.dest_rank(ks[i], world) == owner] for col in (ks, ss, vs)) for ks, ss, vs in cat]
        w1 = play(j, mine)
        j.close()
    finally:
        ctx.close()
    assert w1[0] == CAPACITY, w1
    assert results[owner] == w1
    want = po.run_join(cat, im, em)
    for r in range(world):
        if r != owner:
            owned = [[row for row in rows if po.dest_rank(row[0], world) == r] for rows in want]
            assert results[r] == [(rows, [min(c + 1, 3)] * len(rows)) for c, rows in enumerate(owned)], r
            assert sum(map(len, owned)) == 9


# ---- edges ------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("owner", range(3))
def test_every_row_to_one_owner(owner):
    """At W = 3 every rank sends max_batch_rows rows, all owned by rank `owner`: the owner receives 3 x max_batch_rows
    rows per call."""
    world, B = 3, 4096
    im, em = [("last", "complete"), ("first", "running"), ("last", "final")][owner]
    rnd = random.Random(f"one-owner-3-{owner}")
    keys = _owned_by(owner, world, 700)
    acts = []
    for _ in range(2):
        per_rank = []
        for _ in range(world):
            ks = [rnd.choice(keys) for _ in range(B)]
            per_rank.append((ks, [rnd.randrange(2) for _ in ks], [rnd.randrange(2**64) for _ in ks]))
        acts.append(per_rank)
    out = check_against_one_rank(world, acts, im, em, [1, 2], capacity_hint=1024, max_batch_rows=B, max_emit_rows=world * B)
    assert sum(map(len, out)) > 0


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("im,em", MODES)
def test_zero_and_sentinel_keys(world, im, em):
    """Keys 0 and 2^64-1 (the table's empty marker) with their sides on different ranks, over four calls."""
    rnd = random.Random(f"edge-keys-{world}-{im}-{em}")
    last = world - 1
    # (call, rank): rows (key, side) every world gets, then up to two random ones
    fixed = {(0, 0): [(0, 0)], (0, last): [(SENTINEL, 1)], (1, 1): [(0, 1), (SENTINEL, 0)], (2, last): [(0, 0)],
             (2, 0): [(SENTINEL, 1), (SENTINEL, 0)]}
    acts = []
    for c in range(4):
        per_rank = []
        for r in range(world):
            rows = fixed.get((c, r), []) + [(rnd.choice([0, SENTINEL, 1]), rnd.randrange(2)) for _ in range(rnd.randrange(3))]
            vals = [rnd.choice([0, 2**64 - 1, 2**63, rnd.randrange(2**64)]) for _ in rows]
            per_rank.append(([k for k, _ in rows], [s for _, s in rows], vals))
        acts.append(per_rank)
    out = check_against_one_rank(world, acts, im, em, [1, 1, 4, 6], capacity_hint=16, max_batch_rows=8, max_emit_rows=64)
    assert any(row[0] == 0 for rows in out for row in rows) and any(row[0] == SENTINEL for rows in out for row in rows)
