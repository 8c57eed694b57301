"""What each part of the segment fold's table side is worth on C1 (bench.py's workload: tumbling count over 2^24-row
activations, 10^6 keys): k_segfold's mean CUDA-event time with every part on, with each part switched off in turn
(`WindowFold.set_segfold_parts`, bw_fold_set_segfold_parts), the variants alternating round by round.
Results do not depend on the parts; the counts are checked anyway.  Needs a GPU.

    python tools/bench_segfold_parts.py [--rounds 5] [--steps 32] [--warmup 4]

Prints one JSON line: per variant the per-round means of k_segfold and k_scatter (ms), their median and spread."""

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ALIGN_US = 1_640_995_200_000_000
WINDOW_US = 60_000_000
KEYCOL = 1  # keys from the dense key column (Table::keys) instead of the hot slots
VARIANTS = {"all": KEYCOL, "no_keycol": 0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--batch-rows", type=int, default=1 << 24)
    ap.add_argument("--n-keys", type=int, default=1_000_000)
    args = ap.parse_args()
    os.environ["BW_TIMER_STRIDE"] = "1"  # CUDA events around every activation's kernels, not every 4th
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    B, K, W = args.batch_rows, args.steps, args.warmup
    nbuf = K + W
    dk = [ctx.dev_alloc(B * 8) for _ in range(nbuf)]
    dv = [ctx.dev_alloc(B * 8) for _ in range(nbuf)]

    def make_fold():
        return gpu.WindowFold(ctx, "count", WINDOW_US, None, ALIGN_US, 0, val_dtype="u64", ts_from_value=True,
                              capacity_hint=args.n_keys, max_batch_rows=B, max_emit_rows=max(1 << 20, (K + W + 2) * B // 40),
                              max_late_rows=1 << 16)

    gen = make_fold()
    for s in range(nbuf):
        gen.gen_c1(dk[s], dv[s], s * B, B, args.n_keys)
    gen.sync()
    gen.close()

    res = {v: {"k_segfold": [], "k_scatter": []} for v in VARIANTS}
    for _ in range(args.rounds):
        for name, parts in VARIANTS.items():
            fold = make_fold()
            fold.set_segfold_parts(parts)
            for s in range(W):
                fold.ingest_device(dk[s], dv[s], None, B)
            fold.sync()
            fold.reset_timers()
            for s in range(W, W + K):
                fold.ingest_device(dk[s], dv[s], None, B)
            fold.sync()
            st = fold.stats()
            em, em_eof = fold.advance(), fold.eof()
            fold.close()
            total = int(em.closed_acc.sum()) + int(em_eof.closed_acc.sum())
            if total != nbuf * B or st.combined_folds != K:  # (reset_timers also restarts the fold counters)
                raise SystemExit(f"{name}: counted {total} rows of {nbuf * B}, {st.combined_folds} segment folds of {K}")
            res[name]["k_segfold"].append(st.sum_fold_ms / max(1, st.timed_folds))
            res[name]["k_scatter"].append(st.sum_scatter_ms / max(1, st.scatter_launches))
    for p in dk + dv:
        ctx.dev_free(p)
    ctx.close()
    out = {}
    for name, r in res.items():
        out[name] = {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "rounds": v} for k, v in r.items()}
    print(json.dumps({"workload": f"C1, {B} rows x {K} timed steps per round, {args.n_keys} keys", "variants": out}))


if __name__ == "__main__":
    main()
