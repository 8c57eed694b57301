"""Timing of the windowed join (K8, `bw_jwin_*`) sharded by key over ranks.

Workload: tools/bench_join_window.py's shape per rank.  `join_window` of 2 sides, insert mode last, emit mode final,
10 s tumbling windows, EventClock wait 1 s, frozen system clock, once with `ordered=True` and once with
`ordered=False`.  Each rank holds B rows per activation (--batch-rows, default 2^22) over 10^6 keys drawn uniformly
(seeded per rank), each on a random side.  An activation of all ranks is one stream of W x B rows covering the next 10 s
of event time, rank r holding its r-th contiguous slice: row i of rank r in activation a is stamped
a * 10 s + (r * B + i) * 10 s / (W * B), plus a uniform jitter of +-1 s, and carries handle a * W * B + r * B + i.  The
rank-major concatenation is therefore the time-ordered stream an owner sees in (source rank, source order), and world 1
is tools/bench_join_window.py at B rows.  The columns are generated on the device before timing and fed through
`bw_jwin_apply_device`; each row goes to its key's owner.

Check, before anything is timed: the same join at 2^16 rows per rank over 5 x 10^4 keys, three activations and EOF, is
run sharded and, on each rank, on a world-1 context fed the rank-major concatenation of every rank's columns.  Every
rank's down, meta and late rows of each call must equal the world-1 rows of the keys it owns, in order (late rows
renamed to rows of the concatenation), and its released handles the world-1 handles of those keys; a mismatch exits
non-zero.  After the timed run: the handles released over all ranks equal the rows ingested, there is one down row per
closed window, and every key a rank returns is one it owns.

Timed: a host clock around `bw_jwin_apply_device` and a device synchronise, per timed activation, summed; the maximum
over ranks is reported.  The clock starts once every rank is ready, so that no rank's time includes waiting in the
exchange for a peer still collecting its rows.  The rows of each activation are collected (`bw_jwin_advance`, not
timed) before the next; EOF flushes the rest.

Modes:
    python tools/bench_join_window_ranks.py                              one GPU, world 1 (compare tools/bench_join_window.py)
    torchrun --nproc-per-node G tools/bench_join_window_ranks.py         G GPUs, one rank each (NCCL world, CUDA IPC)
    python tools/bench_join_window_ranks.py --loopback W                 W ranks as threads on ONE GPU

The loopback mode measures the cost the exchange adds to an activation on one card (every rank shares its SMs and
HBM), not multi-GPU scaling.  Prints one JSON line per order (rank 0) with the card's name and power limit as
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
CHECK_KEYS, CHECK_ROWS, CHECK_ACTS = 50_000, 1 << 16, 3
S = 1_000_000
A = 1_640_995_200_000_000
LENGTH = 10 * S


def card(device):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def owners(keys, world):
    """bw_route(key, world) of every key (oracle.pyoracle.dest_rank, vectorised)."""
    z = keys.astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (((z >> np.uint64(32)) * np.uint64(world)) >> np.uint64(32)).astype(np.int64)


class Columns:
    """Rank r's device columns (keys, sides, handles, ts) of activation a, B rows each."""

    def __init__(self, rank, world, b, n_keys, dev):
        import torch

        g = torch.Generator(device=dev).manual_seed(7 + rank)
        self.rank, self.world, self.b = rank, world, b
        self.keys = torch.randint(0, n_keys, (b,), device=dev, generator=g, dtype=torch.int64)
        self.sides = torch.randint(0, 2, (b,), device=dev, generator=g, dtype=torch.uint8)
        offs = (rank * b + torch.arange(b, device=dev, dtype=torch.int64)) * LENGTH // (world * b)
        self.base_ts = offs + torch.randint(-S, S + 1, (b,), device=dev, generator=g, dtype=torch.int64)
        self.ts = torch.empty(b, device=dev, dtype=torch.int64)
        self.handles = torch.empty(b, device=dev, dtype=torch.int64)
        self.row = torch.arange(b, device=dev, dtype=torch.int64)

    def at(self, a):
        import torch

        torch.add(self.base_ts, A + a * LENGTH, out=self.ts)
        torch.add(self.row, a * self.world * self.b + self.rank * self.b, out=self.handles)
        return self.keys.data_ptr(), self.sides.data_ptr(), self.handles.data_ptr(), self.ts.data_ptr()


def make_join(ctx, ordered, b, world, n_keys, shard):
    from bytewax_b200 import gpu

    return gpu.JoinWindow(ctx, "last", "final", ordered, 2, LENGTH, None, A, S, capacity_hint=n_keys // world + n_keys // (8 * world) + 4096,
                          max_windows_per_key=8, max_queued_rows=world * b if ordered else 0, max_batch_rows=b,
                          max_emit_rows=world * b, max_late_rows=world * b, shard_by_key=shard)


def play(j, cols, acts, on_rows, ready=None, sync=None):
    """`acts` activations through apply_device, each collected; returns the seconds spent in the applies."""
    secs = 0.0
    for a, timed in acts:
        ptrs = cols.at(a)
        sync()
        if ready is not None:
            ready()
        t0 = time.perf_counter()
        j.apply_device(*ptrs, cols.b, epoch=a + 1)
        sync()
        if timed:
            secs += time.perf_counter() - t0
        on_rows(j.advance())
    on_rows(j.eof())
    return secs


def rows_of(out, offsets=None):
    """The comparable columns of one call (down, meta, late); late rows named by their row in the rank-major
    concatenation."""
    late_row = out.late_row if offsets is None else offsets[out.late_rank.astype(np.int64)] + out.late_row
    unset = (out.down_mask[:, None] >> np.arange(out.down_handles.shape[1], dtype=np.uint64) & np.uint64(1)) == 0
    handles = np.where(unset, np.uint64(2**64 - 1), out.down_handles)  # the sides that are set
    return ((out.down_key, out.down_window_id, handles, out.down_epoch), (out.meta_key, out.meta_window_id, out.meta_epoch),
            (out.late_key, out.late_window_id, out.late_epoch, out.late_activation, late_row))


def check_rank(ctx, rank, world, device, ordered):
    """The sharded join at the check size against a world-1 join of the concatenation, on this rank's keys.  Returns
    (None when they agree, else a description; the sharded join, which the caller closes once every rank is done)."""
    import torch

    dev = f"cuda:{device}"
    sync = lambda: torch.cuda.synchronize(device)  # noqa: E731
    b, n = CHECK_ROWS, CHECK_ACTS
    j = make_join(ctx, ordered, b, world, CHECK_KEYS, True)
    mine = []
    try:
        play(j, Columns(rank, world, b, CHECK_KEYS, dev), [(a, False) for a in range(n)], mine.append, sync=sync)
    except BaseException:
        j.close()
        raise
    return compare(mine, world_one(world, device, ordered, b, n, sync), rank, world, b), j


def world_one(world, device, ordered, b, n, sync):
    """A world-1 join's rows per call over the rank-major concatenation of every rank's check columns, and the key of
    every handle of an activation."""
    import torch

    from bytewax_b200 import gpu

    dev = f"cuda:{device}"
    all_cols = [Columns(r, world, b, CHECK_KEYS, dev) for r in range(world)]
    key_of = torch.cat([c.keys for c in all_cols]).cpu().numpy()  # handle h: key_of[h % (W * B)]
    ctx1 = gpu.Context(device)
    j1 = make_join(ctx1, ordered, world * b, 1, CHECK_KEYS, False)
    one = []
    try:
        keys1 = torch.cat([c.keys for c in all_cols])
        sides1 = torch.cat([c.sides for c in all_cols])
        for a in range(n):
            ts1 = torch.cat([c.base_ts for c in all_cols]) + (A + a * LENGTH)
            h1 = torch.arange(world * b, device=dev, dtype=torch.int64) + a * world * b
            sync()
            j1.apply_device(keys1.data_ptr(), sides1.data_ptr(), h1.data_ptr(), ts1.data_ptr(), world * b, epoch=a + 1)
            sync()
            one.append(j1.advance())
        one.append(j1.eof())
    finally:
        j1.close()
        ctx1.close()
    return one, key_of


def compare(mine, world1, rank, world, b):
    """None when every call's rows of this rank equal the world-1 rows of the keys it owns, else where they differ."""
    one, key_of = world1
    if len(mine) != len(one):
        return "number of calls"
    offsets = np.arange(world, dtype=np.uint64) * np.uint64(b)
    for i, (m, o) in enumerate(zip(mine, one)):
        for stream, got, want, keys in zip(("down", "meta", "late"), rows_of(m, offsets), rows_of(o), (o.down_key, o.meta_key, o.late_key)):
            own = owners(keys, world) == rank
            for c, (g, w) in enumerate(zip(got, want)):
                if not np.array_equal(g, w[own]):
                    return f"call {i}, {stream} column {c}"
        rel1 = o.released.astype(np.int64)
        rel1 = rel1[owners(key_of[rel1 % (world * b)], world) == rank]
        if not np.array_equal(np.sort(m.released.astype(np.int64)), np.sort(rel1)):
            return f"call {i}, released handles"
    return None


def run_rank(ctx, rank, world, device, args, ordered, ready):
    """One rank's timed job: (seconds of the timed activations, released handles, down rows, meta rows, the keys it
    returned, the join, which the caller closes once every rank is done)."""
    import torch

    b = args.batch_rows
    j = make_join(ctx, ordered, b, world, KEYS, True)
    released = down = meta = 0
    seen = []

    def on_rows(out):
        nonlocal released, down, meta
        released += out.released.size
        down += out.down_key.size
        meta += out.meta_key.size
        seen.append(np.unique(np.concatenate([out.down_key, out.meta_key, out.late_key])))

    try:
        acts = [(a, a >= args.warmup) for a in range(args.warmup + args.steps)]
        secs = play(j, Columns(rank, world, b, KEYS, f"cuda:{device}"), acts, on_rows, ready, lambda: torch.cuda.synchronize(device))
        return secs, released, down, meta, np.unique(np.concatenate(seen)), j
    except BaseException:
        j.close()
        raise


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

    def on_ranks(job):
        """job(ctx, rank, device, ready) on every rank; returns this process's results (all ranks on a loopback world)
        and closes what each job left to close (its last element)."""
        if args.loopback:
            ctxs = gpu.Context.loopback_world(world)
            res, errs = [None] * world, [None] * world
            ready = threading.Barrier(world, timeout=600)

            def body(r):
                try:
                    res[r] = job(ctxs[r], r, 0, ready.wait)
                except BaseException as ex:  # noqa: BLE001 - reported below
                    errs[r] = ex

            threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
            for x in res:
                if x is not None and x[-1] is not None:
                    x[-1].close()
            for c in ctxs:
                c.close()
            for ex in errs:
                if ex is not None:
                    raise ex
            return res
        ctx = gpu.Context(local, rank, world, share_nccl_id(dist, rank, local) if torchrun else None)
        barrier(dist, local)
        x = job(ctx, rank, local, lambda: barrier(dist, local))
        barrier(dist, local)  # no rank destroys its region while a peer may still store into it
        if x[-1] is not None:
            x[-1].close()
        ctx.close()
        return [x]

    def total(v, dtype):
        if dist is None:
            return v
        t = torch.tensor([v], dtype=dtype, device=f"cuda:{local}")
        dist.all_reduce(t, op=dist.ReduceOp.MAX if dtype == torch.float64 else dist.ReduceOp.SUM)
        return t.item()

    mode = "loopback" if args.loopback else "torchrun" if torchrun else "single"
    for ordered in (True, False):
        if world > 1:
            checks = on_ranks(lambda ctx, r, dev, ready: check_rank(ctx, r, world, dev, ordered))
            bad = [(i if args.loopback else rank, c[0]) for i, c in enumerate(checks) if c[0] is not None]
            if total(len(bad), torch.int64):
                raise SystemExit(f"bench_join_window_ranks: WRONG RESULT: rows differ from a world-1 join over the same rows: {bad}")
        res = on_ranks(lambda ctx, r, dev, ready: run_rank(ctx, r, world, dev, args, ordered, ready))
        for i, x in enumerate(res):
            r = i if args.loopback else rank
            if world > 1 and (owners(x[4], world) != r).any():
                raise SystemExit(f"bench_join_window_ranks: WRONG RESULT on rank {r}: a row of a key it does not own")
        secs = total(max(x[0] for x in res), torch.float64)
        released, down, meta = (int(total(sum(x[c] for x in res), torch.int64)) for c in (1, 2, 3))
        ingested = (args.steps + args.warmup) * world * args.batch_rows
        if released != ingested or down != meta:
            raise SystemExit(f"bench_join_window_ranks: WRONG RESULT: released {released} of {ingested} handles; {down} down rows for "
                             f"{meta} closed windows")
        if rank == 0:
            name, power = card(local)
            rows = args.steps * world * args.batch_rows
            print(json.dumps({
                "metric": "events/sec join_window last/final (K8) sharded by key", "value": rows / secs, "unit": "events/s",
                "ordered": ordered, "mode": mode, "ranks": world, "gpus": world if mode == "torchrun" else 1, "steps": args.steps,
                "warmup": args.warmup, "ms_per_step": secs * 1e3 / args.steps, "rows_per_step_per_rank": args.batch_rows, "keys": KEYS,
                "checks": "world > 1: every rank's rows at 2^16 rows per rank == a world-1 join's rows of its keys; handles released "
                          "over all ranks == rows ingested; one down row per closed window; every key on its owner",
                "timing": "host clock around bw_jwin_apply_device + device synchronise from the moment every rank is ready, summed over "
                          "timed steps, max over ranks",
                "card": name, "power_limit": power}), flush=True)
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
