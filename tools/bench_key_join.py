"""Timing of the keyed join (K15, `bw_kjoin_*`) on one GPU.

Three workloads, the columns generated on the device before timing and fed through `bw_kjoin_apply_device`.  Timed:
one activation, `bw_kjoin_apply_device` then `bw_kjoin_advance` (host copies of the rows included), between two CUDA
events; warm-ups, then K timed repetitions, median reported.

1. 2 sides, product, final: 2^24 rows over 10^6 keys drawn uniformly (seeded), each on a random side.  Every repetition
   is a fresh join, so the lists stay at one activation's size (final emits nothing before EOF).  Conservation, after
   the last repetition's EOF: every handle released once, and the rows equal sum over keys of max(1, n_0) * max(1, n_1).
2. 3 sides, last, complete: the same key and side distribution, every repetition one more activation of one join.
   Conservation, after EOF: every handle released once, and the rows equal the emissions counted by a vectorised
   restatement (per key, one emission each time all three sides have been seen since the last one; each is one row).
3. One hot key, last, running, 2 sides: 2^22 rows of key 42 per activation, walked by one thread.  Conservation:
   one row per item, every handle released once.

    python tools/bench_key_join.py [--steps K] [--warmup W]

Prints one JSON line per workload, with the card's name and power limit as `nvidia-smi --query-gpu` reports them during
the same run.
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402  (before libbwgpu: torch loads its own NCCL first)

from bytewax_b200 import gpu  # noqa: E402

ROWS = 1 << 24
KEYS = 1_000_000
HOT_ROWS = 1 << 22


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


class Released:
    """How often each handle of [0, n) came back, counted on the device."""

    def __init__(self, n):
        self.seen = torch.zeros(n, device="cuda", dtype=torch.int32)

    def add(self, out):
        if out.released.size:
            h = torch.from_numpy(out.released.astype("int64")).cuda()
            self.seen.index_add_(0, h, torch.ones(h.numel(), device="cuda", dtype=torch.int32))

    def once(self):
        return bool((self.seen == 1).all())


def timed(j, keys, sides, handles, rows, epoch):
    """One activation, apply_device + advance, between two CUDA events: (seconds, rows out)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    j.apply_device(keys.data_ptr(), sides.data_ptr(), handles.data_ptr(), rows, epoch)
    out = j.advance()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3, out


def columns(seed, n_sides):
    g = torch.Generator(device="cuda").manual_seed(seed)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    sides = torch.randint(0, n_sides, (ROWS,), device="cuda", generator=g, dtype=torch.uint8)
    return keys, sides


def result(name, rows, times, extra):
    times = sorted(times)
    med = times[len(times) // 2]
    return dict({"workload": name, "activation_ms_median": med * 1e3, "rows_per_s": rows / med, "timed_activations": len(times)}, **extra)


def product_final(steps, warmup):
    ctx = gpu.Context(0)
    keys, sides = columns(7, 2)
    handles = torch.arange(ROWS, device="cuda", dtype=torch.int64)
    times, down, rel = [], 0, Released(ROWS)
    for rep in range(warmup + steps):
        j = gpu.KeyJoin(ctx, "product", "final", 2, capacity_hint=KEYS, max_batch_rows=ROWS, max_emit_rows=KEYS, max_product_rows=1 << 27)
        t, out = timed(j, keys, sides, handles, ROWS, 1)
        if rep >= warmup:
            times.append(t)
        if rep == warmup + steps - 1:
            rel.add(out)
            down += out.key.size
            out = j.eof()
            rel.add(out)
            down += out.key.size
        j.close()
    ctx.close()
    n = torch.zeros((KEYS, 2), device="cuda", dtype=torch.int64)
    n.index_put_((keys, sides.to(torch.int64)), torch.ones(ROWS, device="cuda", dtype=torch.int64), accumulate=True)
    want = int(n[n.sum(1) > 0].clamp(min=1).prod(1).sum())
    ok = rel.once() and down == want
    return result("join product/final, 2 sides, 2^24 rows x 10^6 keys per activation, fresh join per activation", ROWS, times,
                  {"down_rows_at_eof": down, "down_rows_expected": want, "every_handle_released_once": rel.once(),
                   "conservation_ok": ok})


def last_complete(steps, warmup):
    ctx = gpu.Context(0)
    n_act = warmup + steps
    keys, sides = columns(11, 3)
    j = gpu.KeyJoin(ctx, "last", "complete", 3, capacity_hint=KEYS, max_batch_rows=ROWS, max_emit_rows=1 << 23, max_product_rows=1 << 24)
    times, down, rel = [], 0, Released(ROWS * n_act)
    perm_g = torch.Generator(device="cuda").manual_seed(13)
    all_keys, all_sides = [], []
    for a in range(n_act):
        p = torch.randperm(ROWS, device="cuda", generator=perm_g)  # each activation: the rows in another order
        k, s = keys[p].contiguous(), sides[p].contiguous()
        all_keys.append(k)
        all_sides.append(s)
        handles = torch.arange(a * ROWS, (a + 1) * ROWS, device="cuda", dtype=torch.int64)
        t, out = timed(j, k, s, handles, ROWS, a + 1)
        if a >= warmup:
            times.append(t)
        rel.add(out)
        down += out.key.size
    out = j.eof()
    rel.add(out)
    down += out.key.size
    j.close()
    ctx.close()
    # per key in arrival order: one emission (one row: each list holds one value) whenever all three sides were seen
    k, s = torch.cat(all_keys), torch.cat(all_sides).to(torch.int64)
    order = torch.sort(k, stable=True).indices
    k, s = k[order], s[order]
    starts = torch.searchsorted(k, torch.arange(KEYS, device="cuda", dtype=torch.int64))
    pos = torch.arange(k.numel(), device="cuda", dtype=torch.int64) - starts[k]
    width = int(pos.max()) + 1
    grid = torch.full((KEYS, width), -1, device="cuda", dtype=torch.int64)
    grid[k, pos] = s
    mask = torch.zeros(KEYS, device="cuda", dtype=torch.int64)
    want = 0
    for c in range(width):
        col = grid[:, c]
        mask = torch.where(col >= 0, mask | torch.bitwise_left_shift(torch.ones_like(col), col.clamp(min=0)), mask)
        full = mask == 7
        want += int(full.sum())
        mask = torch.where(full, torch.zeros_like(mask), mask)
    ok = rel.once() and down == want
    return result("join last/complete, 3 sides, 2^24 rows x 10^6 keys per activation, one join", ROWS, times,
                  {"down_rows": down, "down_rows_expected": want, "every_handle_released_once": rel.once(), "conservation_ok": ok})


def hot_running(steps, warmup):
    ctx = gpu.Context(0)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(17)
    keys = torch.full((HOT_ROWS,), 42, device="cuda", dtype=torch.int64)
    sides = torch.randint(0, 2, (HOT_ROWS,), device="cuda", generator=g, dtype=torch.uint8)
    j = gpu.KeyJoin(ctx, "last", "running", 2, capacity_hint=16, max_batch_rows=HOT_ROWS, max_emit_rows=HOT_ROWS,
                    max_product_rows=HOT_ROWS)
    times, down, rel = [], 0, Released(HOT_ROWS * n_act)
    for a in range(n_act):
        handles = torch.arange(a * HOT_ROWS, (a + 1) * HOT_ROWS, device="cuda", dtype=torch.int64)
        t, out = timed(j, keys, sides, handles, HOT_ROWS, a + 1)
        if a >= warmup:
            times.append(t)
        rel.add(out)
        down += out.key.size
    out = j.eof()
    rel.add(out)
    down += out.key.size
    j.close()
    ctx.close()
    ok = rel.once() and down == HOT_ROWS * n_act
    return result("join last/running, 2 sides, one hot key, 2^22 rows per activation", HOT_ROWS, times,
                  {"down_rows": down, "down_rows_expected": HOT_ROWS * n_act, "every_handle_released_once": rel.once(),
                   "conservation_ok": ok})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    ok = True
    for fn in (product_final, last_complete, hot_running):
        res = fn(args.steps, args.warmup)
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)
        ok = ok and res["conservation_ok"]
    if not ok:
        print("conservation failed", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
