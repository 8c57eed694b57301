"""The claim the sharded keyed join (K6 on N ranks, include/bwgpu.h) rests on: its state is key-local.  Split every
activation of the golden join cases and of seeded streams by owning rank (`po.dest_rank`), run the join restatement
(`po.run_join`) once per owner over its own rows, and the rows of every activation, merged and stably sorted by key
string, are the reference's rows for the whole stream; every row sits on its key's owner."""

import json
import os
import random

import pytest

from oracle import pyoracle as po

WORLDS = [2, 3, 4]
MODES = [(im, em) for im in ("first", "last") for em in ("complete", "final", "running")]
SENTINEL = 2**64 - 1

with open(os.path.join(os.path.dirname(__file__), "golden", "keyed_cases.json")) as _f:
    GOLDEN = json.load(_f)["join"]


def by_owner(batches, world):
    """One stream per rank: each activation keeps the rows that rank owns (possibly none), in source order."""
    out = [[] for _ in range(world)]
    for keys, sides, vals in batches:
        for r in range(world):
            idx = [i for i, k in enumerate(keys) if po.dest_rank(int(k), world) == r]
            out[r].append(([keys[i] for i in idx], [sides[i] for i in idx], [vals[i] for i in idx]))
    return out


def run_sharded(batches, world, im, em):
    """Per activation (then eof): every owner's rows, merged and stably sorted by key string."""
    per_rank = [po.run_join(b, im, em) for b in by_owner(batches, world)]
    merged = []
    for i in range(len(batches) + 1):
        for r in range(world):
            assert all(po.dest_rank(k, world) == r for k, _, _ in per_rank[r][i]), (r, i)
        merged.append(sorted(sum((per_rank[r][i] for r in range(world)), []), key=lambda row: po.key_str(row[0])))
    return merged


def _items(case):
    return [([k], [s], [v]) for k, s, v in case["items"]]


def _cut(case, size):
    items = case["items"]
    return [tuple([it[c] for it in items[a:a + size]] for c in range(3)) for a in range(0, len(items), size)]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("case", range(len(GOLDEN)))
def test_golden_case_sharded(case, world):
    """One item per activation, as the golden plays it: the merged rows are the golden rows, row for row."""
    c = GOLDEN[case]
    got = run_sharded(_items(c), world, c["insert_mode"], c["emit_mode"])
    assert [list(row) for rows in got for row in rows] == c["rows"]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("case", range(len(GOLDEN)))
def test_golden_items_in_activations_sharded(case, world):
    """The golden items in activations of 25: the merged rows are `po.run_join` of the whole stream."""
    c = GOLDEN[case]
    batches = _cut(c, 25)
    assert run_sharded(batches, world, c["insert_mode"], c["emit_mode"]) == po.run_join(batches, c["insert_mode"], c["emit_mode"])


def seeded_stream(seed, n_act=6, n=300, n_keys=80):
    """Activations of up to n rows over n_keys keys (0 and 2^64-1 among them), some of them empty."""
    rnd = random.Random(seed)
    pool = [0, SENTINEL] + [rnd.randrange(1, 2**64 - 1) for _ in range(n_keys // 2)] + [rnd.randrange(1000) for _ in range(n_keys // 2)]
    out = []
    for a in range(n_act):
        m = 0 if a % 4 == 2 else rnd.randrange(1, n)
        ks = [rnd.choice(pool) for _ in range(m)]
        out.append((ks, [rnd.randrange(2) for _ in ks], [rnd.randrange(2**64) for _ in ks]))
    return out


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("im,em", MODES)
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_seeded_stream_sharded(seed, im, em, world):
    batches = seeded_stream(f"join-ranks-{seed}")
    want = po.run_join(batches, im, em)
    assert run_sharded(batches, world, im, em) == want
    assert sum(map(len, want)) > 50


def test_streams_really_shard():
    """Not vacuous: the golden and the seeded streams' keys spread over more than one owner at every world size."""
    for world in WORLDS:
        for c in GOLDEN:
            assert len({po.dest_rank(int(k), world) for k, _, _ in c["items"]}) > 1, world
        keys = {k for seed in (1, 2, 3) for ks, _, _ in seeded_stream(f"join-ranks-{seed}") for k in ks}
        assert len({po.dest_rank(k, world) for k in keys}) == world
