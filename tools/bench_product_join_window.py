"""Timing of the windowed product join (K14, `bw_pjwin_*`) on one GPU.

Two workloads, both `join_window(insert_mode="product")` with 2 sides and emit mode final, the columns generated on the
device before timing and fed through `bw_pjwin_apply_device`; two warm-ups, then K timed repetitions, median reported.

1. Many small windows: 10 s tumbling windows, EventClock wait 1 s, frozen system clock, ordered.  Each activation holds
   2^24 rows over 10^6 keys drawn uniformly (seeded), each on a random side, covering the next 10 s of event time with
   a +-1 s jitter (as tools/bench_join_window.py).  Timed: the activation (`apply_device` to a device synchronise) and,
   separately, the advance that expands the closed windows' products and hands them out (`advance`, host copies
   included).  Conservation, on the device: every handle is released exactly once, and the down rows number
   sum over closed windows of max(1, n_0) * max(1, n_1), n_s counted from the on-time input.
2. A hot window: one key, 2^11 values per side in one window.  Timed: `k_pjwin_expand` alone (its device time as
   `torch.profiler` reports the kernel), as rows/s and as bytes written (8 columns of 8 bytes per row) over 3.35 TB/s,
   the H100 SXM's HBM3 peak.  Conservation: 2^22 rows in `itertools.product` order, every handle released once.

    python tools/bench_product_join_window.py [--steps K] [--warmup W]

Prints one JSON line per workload, with the card's name and power limit as `nvidia-smi --query-gpu` reports them during
the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402  (before libbwgpu: torch loads its own NCCL first)

from bytewax_b200 import gpu  # noqa: E402

ROWS = 1 << 24
KEYS = 1_000_000
S = 1_000_000
A = 1_640_995_200_000_000
LENGTH = 10 * S
HBM_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def many_windows(steps, warmup):
    ctx = gpu.Context(0)
    j = gpu.ProductJoinWindow(ctx, "final", True, 2, LENGTH, None, A, S, capacity_hint=KEYS, max_windows_per_key=8, max_queued_rows=ROWS,
                              max_batch_rows=ROWS, max_emit_rows=ROWS, max_late_rows=ROWS, max_product_rows=1 << 29)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    sides = torch.randint(0, 2, (ROWS,), device="cuda", generator=g, dtype=torch.uint8)
    offs = torch.arange(ROWS, device="cuda", dtype=torch.int64) * LENGTH // ROWS
    jitter = torch.randint(-S, S + 1, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    base_ts = offs + jitter  # handle h: key keys[h % ROWS], side sides[h % ROWS], ts A + base_ts[h % ROWS] + (h // ROWS) * 10 s
    ts = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    handles = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    seen = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.int32)
    late = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.bool)
    down = meta = 0
    t_apply, t_adv = [], []

    def collect(out, a):
        nonlocal down, meta
        down += out.down_key.size
        meta += out.meta_key.size
        if out.released.size:
            seen.index_add_(0, torch.from_numpy(out.released.astype("int64")).cuda(), torch.ones(out.released.size, device="cuda", dtype=torch.int32))
        if out.late_key.size:
            h = torch.from_numpy(out.late_activation.astype("int64") * ROWS + out.late_row.astype("int64")).cuda()
            late[h] = True

    for a in range(n_act):
        torch.add(base_ts, A + a * LENGTH, out=ts)
        torch.add(torch.arange(ROWS, device="cuda", dtype=torch.int64), a * ROWS, out=handles)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        j.apply_device(keys.data_ptr(), sides.data_ptr(), handles.data_ptr(), ts.data_ptr(), ROWS, epoch=a + 1)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        out = j.advance()
        t2 = time.perf_counter()
        if a >= warmup:
            t_apply.append(t1 - t0)
            t_adv.append(t2 - t1)
        collect(out, a)
    collect(j.eof(), n_act)
    j.close()
    ctx.close()
    # the expected row count: per (key, window) of the on-time input, max(1, n_0) * max(1, n_1)
    h = torch.arange(ROWS * n_act, device="cuda", dtype=torch.int64)
    on = ~late
    k, s = keys[h % ROWS][on], sides[h % ROWS][on].to(torch.int64)
    w = torch.div(A + base_ts[h % ROWS] + (h // ROWS) * LENGTH - A, LENGTH, rounding_mode="floor")[on]
    cell = (k * (4 * n_act + 8) + (w + 4)) * 2 + s
    u, c = torch.unique(cell, return_counts=True)
    win, side = torch.div(u, 2, rounding_mode="floor"), u % 2
    n = torch.zeros((int(win.max()) + 1 if win.numel() else 1, 2), device="cuda", dtype=torch.int64)
    n[win, side] = c
    present = (n.sum(1) > 0)
    want = int((n[present].clamp(min=1).prod(1)).sum())
    released_once = bool((seen == 1).all())
    t_apply.sort()
    t_adv.sort()
    return {
        "workload": "join_window product/final, 2 sides, tumbling 10 s, wait 1 s, ordered, 2^24 rows x 10^6 keys per activation",
        "events_per_s": ROWS * len(t_apply) / sum(t_apply),
        "activation_ms_median": t_apply[len(t_apply) // 2] * 1e3,
        "advance_ms_median": t_adv[len(t_adv) // 2] * 1e3,
        "timed_activations": len(t_apply),
        "rows_ingested": ROWS * n_act,
        "down_rows": down,
        "down_rows_expected": want,
        "meta_rows": meta,
        "late_rows": int(late.sum()),
        "every_handle_released_once": released_once,
        "conservation_ok": released_once and down == want and meta == int(present.sum()),
    }


def hot_window(steps, warmup):
    from torch.profiler import ProfilerActivity, profile

    n = 1 << 11
    ctx = gpu.Context(0)
    rnd = np.random.default_rng(5)
    side_np = rnd.permutation(np.repeat(np.arange(2, dtype=np.uint8), n))
    vals_np = rnd.permutation(np.arange(2 * n, dtype=np.uint64))
    keys = torch.full((2 * n,), 7, device="cuda", dtype=torch.int64)
    sides = torch.from_numpy(side_np).cuda()
    vals = torch.from_numpy(vals_np.view(np.int64)).cuda()
    ts = torch.full((2 * n,), A, device="cuda", dtype=torch.int64) + torch.arange(2 * n, device="cuda")
    times, ok = [], True
    for rep in range(warmup + steps):
        j = gpu.ProductJoinWindow(ctx, "final", False, 2, LENGTH, None, A, S, capacity_hint=16, max_windows_per_key=4,
                                  max_batch_rows=2 * n, max_product_rows=n * n)
        torch.cuda.synchronize()
        j.apply_device(keys.data_ptr(), sides.data_ptr(), vals.data_ptr(), ts.data_ptr(), 2 * n)
        assert j.advance().down_key.size == 0
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = j.eof()
            torch.cuda.synchronize()
        us = sum(e.device_time for e in prof.events() if "k_pjwin_expand" in e.name)
        if rep >= warmup:
            times.append(us * 1e-6)
        if rep == warmup:  # checked once: the order is the same on every repetition
            l0, l1 = vals_np[side_np == 0], vals_np[side_np == 1]
            ok = (out.down_key.size == n * n and np.array_equal(out.down_handles[:, 0], np.repeat(l0, n))
                  and np.array_equal(out.down_handles[:, 1], np.tile(l1, n)) and sorted(out.released.tolist()) == list(range(2 * n)))
        j.close()
    ctx.close()
    times.sort()
    med = times[len(times) // 2]
    rows = n * n
    return {
        "workload": "join_window product/final, one key, one window, 2 sides x 2^11 values: k_pjwin_expand alone",
        "expand_us_median": med * 1e6,
        "rows": rows,
        "rows_per_s": rows / med,
        "bytes_written": rows * 64,
        "fraction_of_3_35_TBps": rows * 64 / med / HBM_BPS,
        "timed_repetitions": len(times),
        "conservation_ok": bool(ok),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    ok = True
    for fn in (many_windows, hot_window):
        res = fn(args.steps, args.warmup)
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)
        ok = ok and res["conservation_ok"]
    if not ok:
        print("conservation failed", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
