"""Timing of the keyed collect (K13, `bw_kcollect_*`) on one GPU, and of the host engine on the same flow.

Device workloads, each activation one `bw_kcollect_apply_device` of 2^22 rows followed by `bw_kcollect_advance` at a
system time that lets no timeout fire (so every list is cut by size):
  - `spread`: keys drawn uniformly (seeded) from 10^5, at max_size 64 and at max_size 4096;
  - `hot`: every row of one key, at max_size 10^6.
Row i of activation a carries handle a * 2^22 + i.  The columns are generated on the device before timing.  Two
warm-up activations, then K timed ones; CUDA events bracket apply + advance (the advance copies the lists to the host,
so it ends in a device synchronise).  Conservation is checked at the end: every handle comes back exactly once, after
EOF.

Host: `run_main` of `collect` (max_size 64, 10^3 keys) over 2^17 items, the same flow with `gpu=False` and `gpu=True`,
each timed end to end with a host clock.

    python tools/bench_key_collect.py [--steps K] [--warmup W]

Prints one JSON line per configuration with rows/s, the median activation time, and the card's name and power limit as
`nvidia-smi --query-gpu` reports them during the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import time
from datetime import timedelta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402  (before libbwgpu: torch loads its own NCCL first)

from bytewax_b200 import gpu  # noqa: E402

ROWS = 1 << 22
T0 = 1_700_000_000 * 1_000_000


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def run_device(name, n_keys, max_size, steps, warmup):
    ctx = gpu.Context(0)
    c = gpu.KeyCollect(ctx, max_size, capacity_hint=max(n_keys, 1), max_batch_rows=ROWS, max_emit_rows=ROWS)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(5)
    keys = [torch.randint(0, n_keys, (ROWS,), device="cuda", generator=g, dtype=torch.int64) for _ in range(n_act)]
    handles = [torch.arange(a * ROWS, (a + 1) * ROWS, device="cuda", dtype=torch.int64) for a in range(n_act)]
    seen = torch.zeros(n_act * ROWS, dtype=torch.int32)
    times, emitted = [], 0

    def count(out):
        idx = torch.from_numpy(out.handle.view("int64"))
        seen.index_add_(0, idx, torch.ones_like(idx, dtype=torch.int32))

    try:
        for a in range(n_act):
            b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            b.record()
            c.apply_device(keys[a].data_ptr(), handles[a].data_ptr(), ROWS, a + 1, T0 + 10**12)
            out = c.advance(T0)
            e.record()
            e.synchronize()
            count(out)
            if a >= warmup:
                times.append(b.elapsed_time(e))
                emitted += out.handle.size
        count(c.eof())
    finally:
        c.close()
        ctx.close()
    assert bool((seen == 1).all()), "a handle was lost or emitted twice"
    times.sort()
    total = sum(times) / 1e3
    return dict(config=name, keys=n_keys, max_size=max_size, rows_per_activation=ROWS, activations=steps,
                rows_per_s=steps * ROWS / total, median_ms=times[len(times) // 2], handles_emitted_per_s=emitted / total)


def run_host(use_gpu, n=1 << 17, n_keys=1000):
    import bytewax_b200.operators as op
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource, run_main

    items = [(str(i * 7919 % n_keys), i) for i in range(n)]
    out = []
    flow = Dataflow("bench")
    s = op.input("in", flow, TestingSource(items, batch_size=1 << 14))
    s = op.key_on("key", s, lambda x: x[0])
    op.output("out", op.collect("collect", s, timedelta(seconds=60), 64), TestingSink(out))
    t = time.perf_counter()
    run_main(flow, gpu=use_gpu)
    dt = time.perf_counter() - t
    assert sum(len(v) for _k, v in out) == n
    return dict(config="engine_gpu" if use_gpu else "engine_host", items=n, keys=n_keys, max_size=64, items_per_s=n / dt, seconds=dt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    results = [run_device("spread", 100_000, 64, args.steps, args.warmup), run_device("spread", 100_000, 4096, args.steps, args.warmup),
               run_device("hot", 1, 1_000_000, args.steps, args.warmup), run_host(False), run_host(True)]
    for res in results:
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
