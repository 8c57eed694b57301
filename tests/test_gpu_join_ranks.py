"""K6, the two-sided keyed join, sharded by key over W ranks: threads of one process on a loopback world (include/bwgpu.h,
bw_loopback_create), whose partition kernels, peer stores into the owners' receive regions and barriers are the ones an
NCCL world runs.  -m gpu.

Each rank applies its own rows per activation; each row goes to rank `po.dest_rank(key, W)`, which joins what arrived in
(source rank, source order).  The rows of all ranks, merged and stably sorted by (epoch, key string), must equal row for
row what `po.run_join` and a world-1 `KeyedJoin` give for the rank-major concatenation of every rank's columns."""

import random
import threading

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po  # checker only

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
SENTINEL = 2**64 - 1  # the key table's empty marker; the key itself lives in the alias slot `cap`
MODES = [(im, em) for im in ("first", "last") for em in ("complete", "final", "running")]


def run_ranks(world, body):
    """body(rank, ctx, keep) on one thread per rank of a loopback world.  Joins appended to `keep` are closed only once
    every rank is done, since peers store into each other's regions.  Returns (results, errors), one of each per rank."""
    from bytewax_b200 import gpu

    ctxs = gpu.Context.loopback_world(world)
    results, errors, keep = [None] * world, [None] * world, [[] for _ in range(world)]

    def main(r):
        try:
            results[r] = body(r, ctxs[r], keep[r])
        except BaseException as ex:  # noqa: BLE001 - reported by the caller
            errors[r] = ex

    threads = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for js in keep:
        for j in js:
            j.close()
    for c in ctxs:
        c.close()
    return results, errors


def no_errors(errors):
    for ex in errors:
        if ex is not None:
            raise ex


def arrays(k, s, v):
    return np.array(k, np.uint64), np.array(s, np.uint8), np.array(v, np.uint64)


def concat(per_rank):
    """The rank-major concatenation of one activation's columns."""
    return tuple(sum((list(p[c]) for p in per_rank), []) for c in range(3))


def merged(per_rank_rows):
    """Every rank's rows of one activation (or of eof), stably sorted by key string."""
    return sorted(sum(per_rank_rows, []), key=lambda row: str(row[0]))


def join_ranks(world, acts, im, em, epochs, **kw):
    """Every rank applies its slice of each activation and advances, then eofs.  Per rank: a list of row lists (one per
    activation, then eof) and the epochs of those rows."""
    from bytewax_b200 import gpu

    def body(r, ctx, keep):
        j = gpu.KeyedJoin(ctx, im, em, **kw)
        keep.append(j)
        out, eps = [], []
        for per_rank, e in zip(acts, epochs):
            j.apply(*arrays(*per_rank[r]), epoch=e)
            rows, ep = j.advance()
            out.append(rows)
            eps.append(ep.tolist())
        rows, ep = j.eof()
        return out + [rows], eps + [ep.tolist()]

    results, errors = run_ranks(world, body)
    no_errors(errors)
    return results


def one_rank(acts, im, em, epochs, **kw):
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    j = gpu.KeyedJoin(ctx, im, em, **kw)
    out = []
    for per_rank, e in zip(acts, epochs):
        j.apply(*arrays(*concat(per_rank)), epoch=e)
        out.append(j.advance()[0])
    out.append(j.eof()[0])
    j.close()
    ctx.close()
    return out


def check_against_one_rank(world, acts, im, em, epochs, **kw):
    """Merged rows == po.run_join == world-1 KeyedJoin over the concatenation, per activation and at eof; every rank emits
    only keys it owns, with the activation's epoch.  Returns the merged rows."""
    got = join_ranks(world, acts, im, em, epochs, **kw)
    want = po.run_join([concat(per_rank) for per_rank in acts], im, em)
    w1 = one_rank(acts, im, em, epochs, **dict(kw, max_batch_rows=kw["max_batch_rows"] * world))
    out = []
    for i in range(len(acts) + 1):
        rows = merged([got[r][0][i] for r in range(world)])
        assert rows == want[i] == w1[i], (world, im, em, i)
        out.append(rows)
    for r in range(world):
        for i, rows in enumerate(got[r][0]):
            assert all(po.dest_rank(k, world) == r for k, _, _ in rows), (r, i)
            assert got[r][1][i] == [list(epochs)[min(i, len(epochs) - 1)]] * len(rows), (r, i)
    return out


def streams(world, seed, n_act=6, n=1500, n_keys=400):
    """Seeded activations [per rank (keys, sides, vals)]: keys repeat within and across ranks, include 0 and the
    sentinel, and some ranks have empty activations."""
    rnd = random.Random(seed)
    pool = [0, SENTINEL] + [rnd.randrange(1, SENTINEL) for _ in range(n_keys // 2)] + [rnd.randrange(10**6) for _ in range(n_keys // 2)]
    acts = []
    for a in range(n_act):
        per_rank = []
        for r in range(world):
            m = 0 if (a + r) % 4 == 1 else rnd.randrange(n // 2, n)
            ks = [rnd.choice(pool) for _ in range(m)]
            per_rank.append((ks, [rnd.randrange(2) for _ in ks], [rnd.randrange(2**64) for _ in ks]))
        acts.append(per_rank)
    return acts


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("im,em", MODES)
def test_join_ranks_match_one_rank(world, im, em):
    acts = streams(world, f"ranks-{world}-{im}-{em}")
    assert any(not per_rank[r][0] for per_rank in acts for r in range(world))  # some ranks sit activations out
    epochs = [3 + 2 * i for i in range(len(acts))]
    out = check_against_one_rank(world, acts, im, em, epochs, capacity_hint=1024, max_batch_rows=2048, max_emit_rows=1 << 15)
    assert sum(map(len, out)) > 300  # not vacuous (final: one row per key at eof)


def _owned_by(rank, world, n, start=1):
    out, k = [], start
    while len(out) < n:
        if po.dest_rank(k, world) == rank:
            out.append(k)
        k += 1
    return out


@pytest.mark.parametrize("im,em", [("last", "complete"), ("first", "running"), ("last", "final")])
def test_join_ranks_every_row_to_one_owner(im, em):
    """Every rank sends max_batch_rows rows, all owned by rank 0: the owner receives world x max_batch_rows rows."""
    world, B = 4, 4096
    rnd = random.Random(f"one-owner-{im}-{em}")
    keys = _owned_by(0, world, 700)
    acts = []
    for _ in range(2):
        per_rank = []
        for r in range(world):
            ks = [rnd.choice(keys) for _ in range(B)]
            per_rank.append((ks, [rnd.randrange(2) for _ in ks], [rnd.randrange(2**64) for _ in ks]))
        acts.append(per_rank)
    out = check_against_one_rank(world, acts, im, em, [1, 2], capacity_hint=1024, max_batch_rows=B, max_emit_rows=world * B)
    assert sum(map(len, out)) > 0


@pytest.mark.parametrize("im,em", MODES)
def test_join_ranks_zero_and_sentinel_keys(im, em):
    """Keys 0 and 2^64-1 (the table's empty marker) with their sides on different ranks, over three activations."""
    world = 3
    acts = [
        [([0, SENTINEL], [0, 1], [11, 12]), ([SENTINEL], [0], [13]), ([0], [1], [14])],
        [([], [], []), ([0, 0], [0, 1], [2**64 - 1, 0]), ([SENTINEL, SENTINEL], [1, 0], [2**63, 1])],
        [([SENTINEL], [1], [15]), ([], [], []), ([0], [0], [16])],
    ]
    check_against_one_rank(world, acts, im, em, [1, 1, 4], capacity_hint=16, max_batch_rows=8, max_emit_rows=64)


def _per_rank_split(world, items):
    """Deal one activation's items to the ranks round-robin (each rank's share keeps the items' order)."""
    return [tuple(list(c[r::world]) for c in items) for r in range(world)]


@pytest.mark.parametrize("em", ["complete", "running", "final"])
def test_join_ranks_owner_emit_buffer_full(em):
    """max_emit_rows rows on the owner pass; one more raises BW_ERR_CAPACITY on the owner's advance (or eof) only."""
    from bytewax_b200 import gpu

    world, M = 2, 700

    def items(n):
        keys = _owned_by(1, world, n, start=10**18)
        if em == "running":
            return keys, [i & 1 for i in range(n)], list(range(n))
        if em == "complete":
            return keys + keys, [0] * n + [1] * n, list(range(2 * n))
        return keys, [0] * n, list(range(n))

    acts = [_per_rank_split(world, items(M))]
    out = check_against_one_rank(world, acts, "last", em, [1], capacity_hint=2048, max_batch_rows=4096, max_emit_rows=M)
    assert sum(map(len, out)) == M

    acts = [_per_rank_split(world, items(M + 1))]

    def body(r, ctx, keep):
        j = gpu.KeyedJoin(ctx, "last", em, capacity_hint=2048, max_batch_rows=4096, max_emit_rows=M)
        keep.append(j)
        j.apply(*arrays(*acts[0][r]), epoch=1)
        rows, _ = j.advance()
        rows_eof, _ = j.eof()
        return rows + rows_eof

    results, errors = run_ranks(world, body)
    assert results[0] == [] and errors[0] is None
    assert isinstance(errors[1], N.BwError) and errors[1].status == CAPACITY


def test_join_ranks_owner_key_table_full():
    """cap = max(1024, 2 * capacity_hint) distinct keys plus the sentinel fit on the owner; one key more raises
    BW_ERR_CAPACITY on the owner's advance only."""
    from bytewax_b200 import gpu

    world = 2
    rnd = random.Random("ranks-table-full")
    keys = _owned_by(0, world, 1024, start=0)
    if po.dest_rank(SENTINEL, world) == 0:
        keys.append(SENTINEL)
    first = keys + [rnd.choice(keys) for _ in range(500)]
    rnd.shuffle(first)
    acts = [_per_rank_split(world, (first, [rnd.randrange(2) for _ in first], [rnd.randrange(2**64) for _ in first]))]
    check_against_one_rank(world, acts, "last", "running", [1], capacity_hint=16, max_batch_rows=2048, max_emit_rows=4096)

    new = _owned_by(0, world, 1, start=keys[-2] + 1 if keys[-1] == SENTINEL else keys[-1] + 1)[0]

    def body(r, ctx, keep):
        j = gpu.KeyedJoin(ctx, "last", "running", capacity_hint=16, max_batch_rows=2048, max_emit_rows=4096)
        keep.append(j)
        j.apply(*arrays(*acts[0][r]), epoch=1)
        j.advance()
        j.apply(*arrays([new] if r == 1 else [], [0] if r == 1 else [], [5] if r == 1 else []), epoch=2)
        return j.advance()[0]

    results, errors = run_ranks(world, body)
    assert results[1] == [] and errors[1] is None
    assert isinstance(errors[0], N.BwError) and errors[0].status == CAPACITY


def test_join_ranks_epochs_differ():
    """Ranks that pass different epochs to one call: BW_ERR_STATE on every rank, after a call on which they agreed."""
    from bytewax_b200 import gpu

    world = 3

    def body(r, ctx, keep):
        j = gpu.KeyedJoin(ctx, "last", "complete", capacity_hint=64, max_batch_rows=64)
        keep.append(j)
        j.apply(*arrays([r, r + 1], [0, 1], [1, 2]), epoch=5)
        j.apply(*arrays([r], [0], [3]), epoch=6 if r == 2 else 7)
        return "no error"

    results, errors = run_ranks(world, body)
    assert all(isinstance(e, N.BwError) and e.status == STATE for e in errors), (results, errors)


@pytest.mark.parametrize("world,rows", [(2, 1 << 30), (3, 715_827_883), (4, 1 << 29), (8, 1 << 28)])
def test_join_ranks_batch_limit(world, rows):
    """max_batch_rows x world reaching 2^31 is BW_ERR_SPEC at create, on every rank."""
    from bytewax_b200 import gpu

    assert rows * world >= 2**31 and (rows - 1) * world < 2**31

    def body(r, ctx, keep):
        keep.append(gpu.KeyedJoin(ctx, "last", "complete", capacity_hint=64, max_batch_rows=rows))

    _, errors = run_ranks(world, body)
    assert all(isinstance(e, N.BwError) and e.status == SPEC for e in errors), errors


def test_join_ranks_c4_shape():
    """C4 at W = 4: each rank holds slices of two permutations of [0, N) with payloads 3k+1 (left) and 7k+2 (right);
    insert last, emit complete.  Exactly N pairs (k, 3k+1, 7k+2), each on its key's owner."""
    from bytewax_b200 import gpu

    world, n = 4, 1 << 18
    rnd = np.random.default_rng(44)
    left, right = rnd.permutation(n).astype(np.uint64), rnd.permutation(n).astype(np.uint64)
    n_act = 2
    chunk = n // (world * n_act)

    def body(r, ctx, keep):
        j = gpu.KeyedJoin(ctx, "last", "complete", capacity_hint=n // world + (1 << 14), max_batch_rows=2 * chunk, max_emit_rows=n)
        keep.append(j)
        rows = []
        for a in range(n_act):
            lo = (a * world + r) * chunk
            lk, rk = left[lo:lo + chunk], right[lo:lo + chunk]
            keys = np.empty(2 * chunk, np.uint64)
            keys[0::2], keys[1::2] = lk, rk
            sides = np.tile(np.array([0, 1], np.uint8), chunk)
            vals = np.empty(2 * chunk, np.uint64)
            vals[0::2], vals[1::2] = lk * np.uint64(3) + np.uint64(1), rk * np.uint64(7) + np.uint64(2)
            j.apply(keys, sides, vals, epoch=a + 1)
            rows += j.advance()[0]
        assert j.eof()[0] == []
        return rows

    results, errors = run_ranks(world, body)
    no_errors(errors)
    for r, rows in enumerate(results):
        assert all(po.dest_rank(k, world) == r for k, _, _ in rows)
    allrows = sorted(sum(results, []))
    assert len(allrows) == n
    assert allrows == [(k, 3 * k + 1, 7 * k + 2) for k in range(n)]


def test_join_ranks_memory_returned_on_destroy():
    """Create, use and destroy a W = 2 join three times: device memory comes back (regions, mappings, scratch)."""
    acts = streams(2, "ranks-memory", n_act=3)

    def cycle():
        join_ranks(2, acts, "last", "complete", [1, 2, 3], capacity_hint=1 << 14, max_batch_rows=1 << 16, max_emit_rows=1 << 16)

    cycle()  # warm the allocator's pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        cycle()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
