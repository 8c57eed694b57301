"""What the bucket scatter's write-out settings are worth on C1 (bench.py's workload: tumbling count over 2^24-row
activations, 10^6 keys by default): k_scatter's and k_segfold's mean CUDA-event times with the staging settings the
shape picks, and with the write-out cadence (`BW_SC_EVERY`) and the staging depth (`BW_SC_STG`) forced, the variants
alternating round by round.  Results do not depend on the settings; the counts are checked anyway.  Needs a GPU.

    python tools/bench_scatter_parts.py [--rounds 5] [--steps 32] [--warmup 4] [--n-keys 1000000] [--variants shape,every1,...]

Prints one JSON line: the card and its power limit, then per variant the per-round means of k_scatter and k_segfold
(ms), their median and spread."""

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ALIGN_US = 1_640_995_200_000_000
WINDOW_US = 60_000_000
VARIANTS = {
    "shape": {},
    "every1": {"BW_SC_EVERY": "1"},
    "every2": {"BW_SC_EVERY": "2"},
    "every3": {"BW_SC_EVERY": "3"},
    "stg8": {"BW_SC_STG": "8"},
    "stg16": {"BW_SC_STG": "16"},
}
SWITCHES = ("BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--batch-rows", type=int, default=1 << 24)
    ap.add_argument("--n-keys", type=int, default=1_000_000)
    ap.add_argument("--variants", default=",".join(VARIANTS))
    args = ap.parse_args()
    names = args.variants.split(",")
    for n in names:
        if n not in VARIANTS:
            raise SystemExit(f"unknown variant {n!r}: one of {', '.join(VARIANTS)}")
    os.environ["BW_TIMER_STRIDE"] = "1"  # CUDA events around every activation's kernels, not every 4th
    for k in SWITCHES:
        os.environ.pop(k, None)
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

    res = {v: {"k_scatter": [], "k_segfold": []} for v in names}
    for _ in range(args.rounds):
        for name in names:
            env = VARIANTS[name]
            os.environ.update(env)  # read once, when the fold is created
            try:
                fold = make_fold()
            finally:
                for k in env:
                    del os.environ[k]
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
            res[name]["k_scatter"].append(st.sum_scatter_ms / max(1, st.scatter_launches))
            res[name]["k_segfold"].append(st.sum_fold_ms / max(1, st.timed_folds))
    for p in dk + dv:
        ctx.dev_free(p)
    ctx.close()
    out = {}
    for name, r in res.items():
        out[name] = {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "rounds": v} for k, v in r.items()}
    print(json.dumps({"card": card(), "workload": f"C1, {B} rows x {K} timed steps per round, {args.n_keys} keys",
                      "variants": out}))


if __name__ == "__main__":
    main()
