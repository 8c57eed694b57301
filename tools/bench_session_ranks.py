"""Timing of the session-window fold (K7, `bw_session_*`) sharded by key over ranks.

Workload: tools/bench_sessions.py's shape per rank.  Session `count_window`, gap 2 s, EventClock wait 1 s, frozen
system clock, `max_sessions_per_key` 64.  Each rank holds B rows per activation (--batch-rows, default 2^22) over 10^6
keys drawn uniformly (seeded per rank).  An activation of all ranks is one stream of W x B rows covering the next 10 s of
event time, rank r holding its r-th contiguous slice: row i of rank r in activation a is stamped
a * 10 s + (r * B + i) * 10 s / (W * B), plus a uniform jitter of +-1 s.  The rank-major concatenation is therefore the
time-ordered stream an owner sees in (source rank, source order), and world 1 is tools/bench_sessions.py at B rows.
The columns are generated on the device before timing and fed through `bw_session_apply_device`; each row goes to its
key's owner.

Timed: a host clock around `bw_session_apply_device` and a device synchronise, per timed activation, summed; the
maximum over ranks is reported.  The clock starts once every rank is ready, so that no rank's time includes waiting in
the exchange for a peer still collecting its rows.  The rows of each activation are collected (`bw_session_advance`, not timed) before the
next; EOF closes the rest.  Checks: the counts of every closed session plus the late rows, over all ranks, equal the rows
ingested over all ranks; every key a rank returns is one it owns.

Modes:
    python tools/bench_session_ranks.py                                one GPU, world 1 (compare tools/bench_sessions.py)
    torchrun --nproc-per-node G tools/bench_session_ranks.py           G GPUs, one rank each (NCCL world, CUDA IPC)
    python tools/bench_session_ranks.py --loopback W                   W ranks as threads on ONE GPU

The loopback mode measures the cost the exchange adds to an activation on one card (every rank shares its SMs and
HBM), not multi-GPU scaling.  Prints one JSON line (rank 0) with the card's name and power limit as
`nvidia-smi --query-gpu` reports them during the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

KEYS = 1_000_000
S = 1_000_000
A = 1_640_995_200_000_000


def card(device):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def run_rank(ctx, rank, world, device, args, ready):
    """One rank's job: (seconds of the timed activations, closed counts + late rows, the keys it returned, the fold,
    which the caller closes once every rank is done)."""
    import torch

    from bytewax_b200 import gpu

    b = args.batch_rows
    sess = gpu.SessionFold(ctx, "count", 2 * S, 1 * S, capacity_hint=KEYS // world + KEYS // (8 * world) + 4096, max_batch_rows=b,
                           max_emit_rows=b, max_late_rows=b, max_sessions_per_key=64, shard_by_key=True)
    try:
        dev = f"cuda:{device}"
        g = torch.Generator(device=dev).manual_seed(7 + rank)
        keys = torch.randint(0, KEYS, (b,), device=dev, generator=g, dtype=torch.int64)
        offs = (rank * b + torch.arange(b, device=dev, dtype=torch.int64)) * (10 * S) // (world * b)
        jitter = torch.randint(-S, S + 1, (b,), device=dev, generator=g, dtype=torch.int64)
        ts = torch.empty(b, device=dev, dtype=torch.int64)
        secs, conserved, seen = 0.0, 0, []

        def collect(rows):
            nonlocal conserved
            conserved += int(rows.closed_acc.sum()) + rows.late_key.size
            seen.append(np.unique(np.concatenate([rows.closed_key, rows.late_key])))

        for a in range(args.warmup + args.steps):
            torch.add(offs, jitter, out=ts)
            ts.add_(A + a * 10 * S)
            torch.cuda.synchronize(device)
            ready()
            t0 = time.perf_counter()
            sess.apply_device(keys.data_ptr(), None, ts.data_ptr(), b, epoch=a + 1)
            torch.cuda.synchronize(device)
            if a >= args.warmup:
                secs += time.perf_counter() - t0
            collect(sess.advance())
        collect(sess.eof())
        return secs, conserved, np.unique(np.concatenate(seen)), sess
    except BaseException:
        sess.close()
        raise


def check_owner(keys, world, rank):
    from oracle import pyoracle as po  # the routing function, restated

    if world > 1 and any(po.dest_rank(int(k), world) != rank for k in keys.tolist()):
        raise SystemExit(f"bench_session_ranks: WRONG RESULT on rank {rank}: a row of a key it does not own")


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
                res[r] = run_rank(ctxs[r], r, world, 0, args, ready.wait)
            except BaseException as ex:  # noqa: BLE001 - reported below
                errs[r] = ex

        threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for x in res:
            if x is not None:
                x[3].close()
        for c in ctxs:
            c.close()
        for ex in errs:
            if ex is not None:
                raise ex
        for r, x in enumerate(res):
            check_owner(x[2], world, r)
        secs, conserved = max(x[0] for x in res), sum(x[1] for x in res)
    else:
        mode = "torchrun" if torchrun else "single"
        ctx = gpu.Context(local, rank, world, share_nccl_id(dist, rank, local) if torchrun else None)
        barrier(dist, local)
        secs, conserved, seen, sess = run_rank(ctx, rank, world, local, args, lambda: barrier(dist, local))
        barrier(dist, local)  # no rank destroys its region while a peer may still store into it
        sess.close()
        ctx.close()
        check_owner(seen, world, rank)
        if dist is not None:
            t = torch.tensor([secs], dtype=torch.float64, device=f"cuda:{local}")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            secs = float(t.item())
            t = torch.tensor([conserved], dtype=torch.int64, device=f"cuda:{local}")
            dist.all_reduce(t)
            conserved = int(t.item())
            dist.destroy_process_group()
    ingested = (args.steps + args.warmup) * world * args.batch_rows
    if conserved != ingested:
        raise SystemExit(f"bench_session_ranks: WRONG RESULT: closed counts + late rows {conserved} != rows ingested {ingested}")
    if rank == 0:
        name, power = card(local)
        rows = args.steps * world * args.batch_rows
        print(json.dumps({
            "metric": "events/sec session count_window (K7) sharded by key", "value": rows / secs, "unit": "events/s",
            "mode": mode, "ranks": world, "gpus": world if mode == "torchrun" else 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": secs * 1e3 / args.steps, "rows_per_step_per_rank": args.batch_rows, "keys": KEYS,
            "checks": "closed counts + late rows over all ranks == rows ingested; every key on its owner",
            "timing": "host clock around bw_session_apply_device + device synchronise from the moment every rank is ready, summed over "
                      "timed steps, max over ranks",
            "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
