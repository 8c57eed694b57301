"""The claim the sharded z-score map (K5 on N ranks, include/bwgpu.h) rests on: its state is key-local.  Split every
activation of the golden z-score cases and of seeded Zipf streams by owning rank (`po.dest_rank`), run the mapper
(`po.run_zscore`) once per owner over its own rows, put each result back at its row's source position, and the result
is the mapper's over the whole stream, bit for bit."""

import json
import os
import struct

import numpy as np
import pytest

from oracle import pyoracle as po

WORLDS = [2, 3, 4]

with open(os.path.join(os.path.dirname(__file__), "golden", "keyed_cases.json")) as _f:
    GOLDEN = json.load(_f)["zscore"]


def _bits(rows):
    return [(struct.pack("<d", m), struct.pack("<d", s), bool(f)) for m, s, f in rows]


def run_sharded(batches, world, **kw):
    """Per activation, the rows of `batches` mapped by one mapper per owner over the rows it owns, in source order."""
    owners = [[] for _ in range(world)]  # per owner, per activation: (keys, vals, source positions)
    for keys, vals in batches:
        dest = [po.dest_rank(int(k), world) for k in keys]
        for r in range(world):
            idx = [i for i, d in enumerate(dest) if d == r]
            owners[r].append(([keys[i] for i in idx], [vals[i] for i in idx], idx))
    per_owner = [po.run_zscore([(k, v) for k, v, _ in owners[r]], **kw) for r in range(world)]
    out = []
    for a, (keys, _) in enumerate(batches):
        rows = [None] * len(keys)
        for r in range(world):
            for i, row in zip(owners[r][a][2], per_owner[r][a]):
                rows[i] = row
        assert all(row is not None for row in rows)
        out.append(rows)
    return out


def _cut(keys, vals, n_acts):
    cuts = np.linspace(0, len(keys), n_acts + 1).astype(int).tolist()
    return [(keys[cuts[i]:cuts[i + 1]], vals[cuts[i]:cuts[i + 1]]) for i in range(n_acts)]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("case", range(len(GOLDEN)))
@pytest.mark.parametrize("n_acts", [1, 3, 7])
def test_golden_case_sharded(case, world, n_acts):
    c = GOLDEN[case]
    got = run_sharded(_cut(c["keys"], c["vals"], n_acts), world)
    assert [[m, s, f] for rows in got for m, s, f in rows] == c["rows"]


def zipf_stream(seed, n_acts, rows, n_keys=100_000):
    rnd = np.random.default_rng(seed)
    return [(np.minimum(rnd.zipf(1.1, rows), n_keys).tolist(), rnd.normal(0.0, 1.0, rows).astype(np.float32).astype(float).tolist())
            for _ in range(n_acts)]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("window", [1, 10, 32])
def test_zipf_stream_sharded(seed, world, window):
    batches = zipf_stream(seed, 4, 1500)
    for rounded in (False, True):
        kw = dict(window=window, threshold=2.0, correctly_rounded=rounded)
        want = po.run_zscore(batches, **kw)
        got = run_sharded(batches, world, **kw)
        assert [_bits(a) for a in got] == [_bits(a) for a in want]


def test_streams_really_shard():
    """Not vacuous: the golden and the Zipf streams' keys spread over more than one owner at every world size."""
    for world in WORLDS:
        for c in GOLDEN:
            if len(set(c["keys"])) > 4:
                assert len({po.dest_rank(int(k), world) for k in c["keys"]}) > 1, world
        keys = {k for seed in (1, 2, 3) for ks, _ in zipf_stream(seed, 4, 1500) for k in ks}
        assert len({po.dest_rank(int(k), world) for k in keys}) == world
