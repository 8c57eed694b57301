"""The claim the sharded session fold (K7 on N ranks, include/bwgpu.h) rests on: its state is key-local.  Split every
batch of the golden and seeded session streams by owning rank (`po.dest_rank`), run the session restatement
(tests/session_oracle.py) once per owner over its own rows, and the rows of every step, merged and stably sorted by key
string, are the reference's rows for the whole stream."""

import json
import os

import pytest

from oracle import pyoracle as po
from oracle.streams import rows_digest
from tests import session_oracle as so
from tests.test_oracle_sessions import _same

WORLDS = [2, 3, 4]

with open(os.path.join(os.path.dirname(__file__), "golden", "session_cases.json")) as _f:
    GOLDEN = json.load(_f)


def by_owner(steps, world):
    """One stream per rank: each batch keeps the rows that rank owns (possibly none); notify steps go to every rank."""
    out = [[] for _ in range(world)]
    for step in steps:
        if step[0] != "batch":
            for r in range(world):
                out[r].append(step)
            continue
        _, now, keys, ts, vals = step
        for r in range(world):
            idx = [i for i, k in enumerate(keys) if po.dest_rank(int(k), world) == r]
            out[r].append(["batch", now, [keys[i] for i in idx], [ts[i] for i in idx], [vals[i] for i in idx]])
    return out


def run_sharded(spec, steps, world):
    per_rank = [so.run_sessions(spec, s) for s in by_owner(steps, world)]
    merged = []
    for i in range(len(per_rank[0])):
        rows = sum((per_rank[r][i] for r in range(world)), [])
        assert all(po.dest_rank(row[0], world) == r for r in range(world) for row in per_rank[r][i])
        merged.append(sorted(rows, key=lambda row: str(row[0])))
    return merged


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_golden_case_sharded(name, world):
    case = GOLDEN["cases"][name]
    assert _same(run_sharded(case["spec"], case["steps"], world), case["acts"])


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("seed", list(so.SEEDED))
def test_seeded_digest_sharded(seed, world):
    spec, steps = so.seeded_steps(seed, moving=seed % 3 != 0)
    got = run_sharded(spec, steps, world)
    want = GOLDEN["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]


def test_streams_really_shard():
    """Not vacuous: the seeded streams' keys spread over more than one owner at every world size."""
    keys = {k for seed in so.SEEDED for step in so.seeded_steps(seed)[1] if step[0] == "batch" for k in step[2]}
    for world in WORLDS:
        assert len({po.dest_rank(k, world) for k in keys}) > 1, world
