"""Timing of the z-score `stateful_map` (K5, `bw_smap_*`) sharded by key over ranks.

Workload: the C2 shape of `bench.py --config c2` per rank.  Rolling z-score, window 10, threshold 2.0, f32 values drawn
from N(0, 1), keys Zipf-1.1 clipped to 1..10^5.  Each rank holds B rows per activation (--batch-rows, default 2^22,
bench.py's C2 size), generated on the host from a seed per (rank, activation) before timing and passed as HOST columns.
Each row goes to its key's owner; its mu, sigma and flag come back to the rank that passed it.

Zipf-1.1 is skewed: from the distribution, key 1 carries 1 / zeta(1.1) of all rows and the clipped tail, key 10^5,
zeta(1.1, 10^5) / zeta(1.1).  Both shares are printed, with the rows each owner received per activation (from the
routing function over the generated keys), so the load imbalance between owners is visible next to the rate.

Timed: a host clock around `bw_smap_apply` (H2D, exchange, map, return leg, D2H), per timed activation, summed; the
maximum over ranks is reported.  The clock starts once every rank is ready, so that no rank's time includes waiting in
the exchange for a peer still preparing its rows.  Check, before anything is reported: a world-1 map is fed the
rank-major concatenation of every rank's rows, activation by activation, and the SHA-256 of each rank's mu, sigma and
flag bytes must equal that of its slice of the world-1 outputs, for every activation; a mismatch exits non-zero.

Modes:
    python tools/bench_smap_ranks.py                                one GPU, world 1 (compare bench.py --config c2)
    torchrun --nproc-per-node G tools/bench_smap_ranks.py           G GPUs, one rank each (NCCL world, CUDA IPC)
    python tools/bench_smap_ranks.py --loopback W                   W ranks as threads on ONE GPU

The loopback mode measures the cost the exchange adds to an activation on one card (every rank shares its SMs, HBM and
PCIe link), not multi-GPU scaling.  Prints one JSON line (rank 0) with the card's name and power limit as
`nvidia-smi --query-gpu` reports them during the same run.
"""

import argparse
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

KEYS = 100_000
WINDOW, THRESHOLD = 10, 2.0


def card(device):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def columns(rank, act, b):
    rnd = np.random.default_rng([7, rank, act])
    return np.minimum(rnd.zipf(1.1, b), KEYS).astype(np.uint64), rnd.normal(0.0, 1.0, b).astype(np.float32)


def digest(mu, sigma, flag):
    return hashlib.sha256(mu.tobytes() + sigma.tobytes() + flag.tobytes()).hexdigest()


def run_rank(ctx, rank, world, args, ready):
    """One rank's job: (seconds of the timed activations, a digest per activation, the map, which the caller closes once
    every rank is done)."""
    from bytewax_b200 import gpu

    b = args.batch_rows
    cols = [columns(rank, a, b) for a in range(args.warmup + args.steps)]
    zm = gpu.ZScoreMap(ctx, WINDOW, THRESHOLD, "f32", capacity_hint=KEYS, max_batch_rows=b, shard_by_key=world > 1)
    try:
        secs, digests = 0.0, []
        for a, (k, v) in enumerate(cols):
            ready()
            t0 = time.perf_counter()
            out = zm.apply(k, v)
            if a >= args.warmup:
                secs += time.perf_counter() - t0
            digests.append(digest(*out))
        return secs, digests, zm
    except BaseException:
        zm.close()
        raise


def world1_digests(ctx, world, args):
    """Per activation, per rank: the digest of that rank's slice of a world-1 map over the rank-major concatenation."""
    from bytewax_b200 import gpu

    b = args.batch_rows
    zm = gpu.ZScoreMap(ctx, WINDOW, THRESHOLD, "f32", capacity_hint=KEYS, max_batch_rows=b * world)
    try:
        out = []
        for a in range(args.warmup + args.steps):
            cols = [columns(r, a, b) for r in range(world)]
            mu, sigma, flag = zm.apply(np.concatenate([c[0] for c in cols]), np.concatenate([c[1] for c in cols]))
            out.append([digest(mu[r * b:(r + 1) * b], sigma[r * b:(r + 1) * b], flag[r * b:(r + 1) * b]) for r in range(world)])
        return out
    finally:
        zm.close()


def owner_rows(world, args):
    """Rows each owner receives per timed activation, averaged (from the routing function over the generated keys)."""
    from oracle import pyoracle as po  # the routing function, restated

    owner = np.array([po.dest_rank(k, world) for k in range(KEYS + 1)], np.int64)
    tot = np.zeros(world, np.int64)
    for a in range(args.warmup, args.warmup + args.steps):
        for r in range(world):
            tot += np.bincount(owner[columns(r, a, args.batch_rows)[0].astype(np.int64)], minlength=world)
    return (tot // args.steps).tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch-rows", type=int, default=1 << 22, help="rows per rank per activation (B)")
    ap.add_argument("--loopback", type=int, default=0, help="W ranks as threads on one GPU")
    args = ap.parse_args()
    torchrun = int(os.environ.get("WORLD_SIZE", "1")) > 1
    if torchrun and args.loopback:
        raise SystemExit("--loopback runs in one process: not under torchrun")

    from bench import barrier, dist_setup, share_nccl_id  # the rendezvous plumbing bench.py uses

    rank, world, local, dist = dist_setup(0) if torchrun else (0, args.loopback or 1, 0, None)
    import torch  # (before libbwgpu: torch loads its own NCCL first)

    from bytewax_b200 import gpu

    if args.loopback:
        mode = "loopback"
        ctxs = gpu.Context.loopback_world(world)
        res, errs = [None] * world, [None] * world
        ready = threading.Barrier(world, timeout=600)

        def body(r):
            try:
                res[r] = run_rank(ctxs[r], r, world, args, ready.wait)
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
        secs = max(x[0] for x in res)
        mine = {r: x[1] for r, x in enumerate(res)}
        ctx1 = gpu.Context(0)
        want = world1_digests(ctx1, world, args)
        ctx1.close()
    else:
        mode = "torchrun" if torchrun else "single"
        ctx = gpu.Context(local, rank, world, share_nccl_id(dist, rank, local) if torchrun else None)
        barrier(dist, local)
        secs, digests, zm = run_rank(ctx, rank, world, args, lambda: barrier(dist, local))
        barrier(dist, local)  # no rank destroys its region while a peer may still store into it
        zm.close()
        ctx.close()
        mine = {rank: digests}
        ctx1 = gpu.Context(local)
        want = world1_digests(ctx1, world, args)
        ctx1.close()
    bad = [(r, a) for r, ds in mine.items() for a, d in enumerate(ds) if d != want[a][r]]
    if dist is not None:
        t = torch.tensor([secs, len(bad)], dtype=torch.float64, device=f"cuda:{local}")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        secs, n_bad = float(t[0].item()), int(t[1].item())
        dist.destroy_process_group()
    else:
        n_bad = len(bad)
    if n_bad:
        raise SystemExit(f"bench_smap_ranks: WRONG RESULT: outputs differ from a world-1 map over the same rows (rank, activation): {bad[:8]}")
    if rank == 0:
        from scipy.special import zeta

        name, power = card(local)
        rows = args.steps * world * args.batch_rows
        print(json.dumps({
            "metric": "events/sec stateful_map z-score (K5) sharded by key", "value": rows / secs, "unit": "events/s",
            "mode": mode, "ranks": world, "gpus": world if mode == "torchrun" else 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": secs * 1e3 / args.steps, "rows_per_step_per_rank": args.batch_rows, "keys": KEYS,
            "rows_per_owner_per_step": owner_rows(world, args),
            "share_of_rows_key_1": float(1.0 / zeta(1.1)), "share_of_rows_key_1e5_clipped_tail": float(zeta(1.1, KEYS) / zeta(1.1)),
            "checks": "every rank's mu / sigma / flag digest per activation == its slice of a world-1 map over the rank-major concatenation",
            "timing": "host clock around bw_smap_apply (host columns in and out) from the moment every rank is ready, summed over "
                      "timed steps, max over ranks",
            "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
