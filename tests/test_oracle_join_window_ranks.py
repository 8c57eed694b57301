"""The claim the sharded windowed join (K8 on N ranks, include/bwgpu.h) rests on: its state is key-local.  Split every
batch of the golden and seeded join-window streams by owning rank (`po.dest_rank`), run the join restatement
(tests/join_window_oracle.py) once per owner over its own rows, and the rows of every step, merged and stably sorted by
key string, are the reference's rows for the whole stream; the handles the owners release in a step are, together,
the ones one run over the whole stream releases in it."""

import json
import os

import pytest

from oracle import pyoracle as po
from oracle.streams import rows_digest
from tests import join_window_oracle as jo

WORLDS = [2, 3, 4]

with open(os.path.join(os.path.dirname(__file__), "golden", "join_window_cases.json")) as _f:
    GOLDEN = json.load(_f)


def by_owner(steps, world):
    """One stream per rank: each batch keeps the rows that rank owns (possibly none); notify steps go to every rank."""
    out = [[] for _ in range(world)]
    for step in steps:
        if step[0] != "batch":
            for r in range(world):
                out[r].append(step)
            continue
        _, now, keys, ts, sides, vals = step
        for r in range(world):
            idx = [i for i, k in enumerate(keys) if po.dest_rank(int(k), world) == r]
            out[r].append(["batch", now] + [[col[i] for i in idx] for col in (keys, ts, sides, vals)])
    return out


def run_sharded(spec, steps, world):
    """Per step (then EOF): the owners' rows merged and stably sorted by key string, and the union of their releases."""
    per_rank = [jo.run_join_window(spec, s) for s in by_owner(steps, world)]
    merged, released = [], []
    for i in range(len(per_rank[0][0])):
        assert all(po.dest_rank(row[0], world) == r for r in range(world) for row in per_rank[r][0][i])
        rows = sum((per_rank[r][0][i] for r in range(world)), [])
        merged.append(sorted(rows, key=lambda row: str(row[0])))
        rel = [h for r in range(world) for h in per_rank[r][1][i]]
        assert len(rel) == len(set(rel)), "a handle released by two owners"
        released.append(sorted(rel))
    return merged, released


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_golden_case_sharded(name, world):
    case = GOLDEN["cases"][name]
    rows, released = run_sharded(case["spec"], case["steps"], world)
    assert rows == case["acts"]
    assert released == jo.run_join_window(case["spec"], case["steps"])[1]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("seed", list(jo.SEEDED))
def test_seeded_digest_sharded(seed, world):
    spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
    rows, released = run_sharded(spec, steps, world)
    want = GOLDEN["seeded"][f"seed_{seed}"]
    assert [len(a) for a in rows] == want["rows"]
    assert rows_digest(rows) == want["sha256"]
    assert released == jo.run_join_window(spec, steps)[1]


def test_streams_really_shard():
    """Not vacuous: the seeded streams' keys spread over more than one owner at every world size, and so do the keys of
    some golden cases at W = 2."""
    keys = {k for seed in jo.SEEDED for step in jo.seeded_steps(seed)[1] if step[0] == "batch" for k in step[2]}
    for world in WORLDS:
        assert len({po.dest_rank(k, world) for k in keys}) > 1, world
    spread = sum(len({po.dest_rank(int(k), 2) for step in case["steps"] if step[0] == "batch" for k in step[2]}) > 1
                 for case in GOLDEN["cases"].values())
    assert spread > 0
