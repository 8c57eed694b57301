"""Timing of the two-stream keyed join (K6, `bw_join_*`) sharded by key over ranks: the C4 shape.

Workload: the left and the right stream are two seeded permutations of [0, N), N = (steps + warmup) x ranks x B, with
payloads 3k+1 (left) and 7k+2 (right); insert last, emit complete.  In activation s, rank r holds the r-th B-row slice
of step s of both streams, interleaved (left, right, left, ...), 2B rows per rank per activation.  Every key meets its
other side on its owner in this or a later activation, so the whole job emits exactly N pairs (k, 3k+1, 7k+2).

Timed: a host clock around `bw_join_apply` + `bw_join_advance` of each timed activation (host columns in, the rows'
host copies out), summed over the timed steps; the maximum over ranks is reported.  Checks, after EOF: every row a rank
emits is (k, 3k+1, 7k+2) with k < N and owned by that rank, no key twice on a rank, and the pair count summed over all
ranks is N.

Modes:
    python tools/bench_join_ranks.py                                   one GPU, world 1 (compare bench.py --config c4)
    torchrun --nproc-per-node G tools/bench_join_ranks.py              G GPUs, one rank each (NCCL world, CUDA IPC)
    python tools/bench_join_ranks.py --loopback W                      W ranks as threads on ONE GPU

The loopback mode measures the cost the exchange adds to an activation on one card (every rank shares its SMs and
HBM), not multi-GPU scaling.  Prints one JSON line (rank 0) with the card's name and power limit as
`nvidia-smi --query-gpu` reports them during the same run.
"""

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card(device):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def streams(n, seed=4):
    rnd = np.random.default_rng(seed)
    return rnd.permutation(n).astype(np.uint64), rnd.permutation(n).astype(np.uint64)


def activation(left, right, s, r, world, b):
    """Rank r's columns of activation s: its B-row slices of both streams, interleaved."""
    lo = (s * world + r) * b
    lk, rk = left[lo:lo + b], right[lo:lo + b]
    keys = np.empty(2 * b, np.uint64)
    keys[0::2], keys[1::2] = lk, rk
    vals = np.empty(2 * b, np.uint64)
    vals[0::2], vals[1::2] = lk * np.uint64(3) + np.uint64(1), rk * np.uint64(7) + np.uint64(2)
    return keys, np.tile(np.array([0, 1], np.uint8), b), vals


def check_rows(key, left, right, n, world, rank):
    """Every row is (k, 3k+1, 7k+2) with k < n, owned by `rank`, no key twice.  Returns the row count."""
    from oracle import pyoracle as po  # the routing function, restated

    ok = bool((key < np.uint64(n)).all() and (left == key * np.uint64(3) + np.uint64(1)).all()
              and (right == key * np.uint64(7) + np.uint64(2)).all() and np.unique(key).size == key.size)
    if not ok:
        raise SystemExit(f"bench_join_ranks: WRONG RESULT on rank {rank}: a pair is not (k, 3k+1, 7k+2) or a key repeats")
    if world > 1:
        sample = key[:: max(1, key.size // 4096)].tolist()
        if any(po.dest_rank(int(k), world) != rank for k in sample):
            raise SystemExit(f"bench_join_ranks: WRONG RESULT on rank {rank}: a row of a key it does not own")
    return int(key.size)


def run_rank(ctx, rank, world, args, left, right):
    """One rank's job: (seconds of the timed steps, pairs emitted, the join, which the caller closes once every rank is
    done)."""
    from bytewax_b200 import _native as N, gpu

    b, steps, warmup = args.batch_rows, args.steps, args.warmup
    n = left.size
    j = gpu.KeyedJoin(ctx, "last", "complete", capacity_hint=n // world + n // (8 * world) + 4096, max_batch_rows=2 * b,
                      max_emit_rows=2 * b * world)  # an owner receives at most 2B rows from each rank per activation
    cols = [activation(left, right, s, rank, world, b) for s in range(steps + warmup)]
    lib, rows = ctx.lib, N.BwJoinRows()
    got, secs = [], 0.0
    try:
        for s in range(steps + warmup):
            keys, sides, vals = cols[s]
            t0 = time.perf_counter()
            j.apply(keys, sides, vals, epoch=s + 1)
            N.check(lib.bw_join_advance(j.h, C.byref(rows)), ctx.h)
            if s >= warmup:
                secs += time.perf_counter() - t0
            got.append(tuple(np.ctypeslib.as_array(p, shape=(rows.n,)).copy() for p in (rows.key, rows.left, rows.right))
                       if rows.n else ())
        rest = j.eof()[0]
        if rest:
            raise SystemExit(f"bench_join_ranks: WRONG RESULT on rank {rank}: {len(rest)} rows at EOF under emit complete")
        got = [g for g in got if g]
        cat = [np.concatenate([g[c] for g in got]) if got else np.zeros(0, np.uint64) for c in range(3)]
        return secs, check_rows(*cat, n, world, rank), j
    except BaseException:
        j.close()
        raise


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch-rows", type=int, default=1 << 21, help="rows per side per rank per activation (B)")
    ap.add_argument("--loopback", type=int, default=0, help="W ranks as threads on one GPU")
    args = ap.parse_args()
    torchrun = int(os.environ.get("WORLD_SIZE", "1")) > 1
    if torchrun and args.loopback:
        raise SystemExit("--loopback runs in one process: not under torchrun")

    from bench import barrier, dist_setup, share_nccl_id  # the rendezvous plumbing bench.py uses

    rank, world, local, dist = dist_setup(0) if torchrun else (0, args.loopback or 1, 0, None)
    import torch  # noqa: F401  (before libbwgpu: torch loads its own NCCL first)

    from bytewax_b200 import gpu

    n = (args.steps + args.warmup) * world * args.batch_rows
    left, right = streams(n)
    if args.loopback:
        mode = "loopback"
        ctxs = gpu.Context.loopback_world(world)
        res, errs = [None] * world, [None] * world

        def body(r):
            try:
                res[r] = run_rank(ctxs[r], r, world, args, left, right)
            except BaseException as ex:  # noqa: BLE001 - reported below
                errs[r] = ex

        threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for x in res:
            if x is not None:
                x[2].close()
        for c in ctxs:
            c.close()
        for ex in errs:
            if ex is not None:
                raise ex
        secs, pairs = max(x[0] for x in res), sum(x[1] for x in res)
    else:
        mode = "torchrun" if torchrun else "single"
        ctx = gpu.Context(local, rank, world, share_nccl_id(dist, rank, local) if torchrun else None)
        barrier(dist, local)
        secs, pairs, j = run_rank(ctx, rank, world, args, left, right)
        barrier(dist, local)  # no rank destroys its region while a peer may still store into it
        j.close()
        ctx.close()
        if dist is not None:
            t = torch.tensor([secs, float(pairs)], dtype=torch.float64, device=f"cuda:{local}")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            secs = float(t[0].item())
            t = torch.tensor([pairs], dtype=torch.int64, device=f"cuda:{local}")
            dist.all_reduce(t)
            pairs = int(t.item())
            dist.destroy_process_group()
    if pairs != n:
        raise SystemExit(f"bench_join_ranks: WRONG RESULT: {pairs} pairs over all ranks, want {n}")
    if rank == 0:
        name, power = card(local)
        rows = args.steps * world * 2 * args.batch_rows
        print(json.dumps({
            "metric": "events/sec two-stream keyed join (K6) sharded by key", "value": rows / secs, "unit": "events/s",
            "mode": mode, "ranks": world, "gpus": world if mode == "torchrun" else 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": secs * 1e3 / args.steps, "rows_per_step_per_rank": 2 * args.batch_rows, "keys": n, "pairs": pairs,
            "checks": "every pair (k, 3k+1, 7k+2), on its owner, once; pairs over all ranks == keys",
            "timing": "host clock around bw_join_apply + bw_join_advance (HOST columns), summed over timed steps, max over ranks",
            "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
