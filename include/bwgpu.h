/*
 * bwgpu.h -- C ABI of libbwgpu.so: the H100 (sm_90a) windowed-fold hot path.
 *
 * This is the drop-in boundary for ONE path of bytewax v0.21.1: key hash ->
 * partition by destination worker -> worker-to-worker exchange -> per-key
 * windowed state update (SURVEY.md section 8).  The reference has no C ABI; its
 * only FFI is the PyO3 module `bytewax._bytewax` (src/lib.rs:24-32).  The
 * functions below are what a maintainer would bind from the Rust host (or,
 * as this repo does, from Python via ctypes) in place of:
 *
 *   bw_ctx_create / bw_ctx_destroy
 *       worker start-up: src/worker.rs:100-159 (`worker_main`), and the
 *       Timely communication set-up src/run.rs:262-274 (`CommunicationConfig`)
 *       -- here one rank per GPU, an NCCL communicator over NVLink and CUDA
 *       IPC mappings of every peer's receive buffers.
 *   bw_route
 *       `PartitionFn::assign` + `PartitionOp::partition`
 *       src/timely.rs:455-465, 494-569 (hash % workers; the hash itself is
 *       un-pinned by the reference, SURVEY.md section 8c).
 *   bw_fold_create / bw_fold_destroy
 *       construction of `StatefulBatchOp::stateful_batch` for a windowed
 *       numeric fold: src/operators.rs:549-660, with the logic builder of
 *       pysrc/bytewax/operators/windowing.py:1254-1319 (`window`) and
 *       :1717-1846 (`fold_window`), clock :365-420 (`EventClock`), windower
 *       :842-926 (`SlidingWindower` / `TumblingWindower`).
 *   bw_ingest_acquire / bw_ingest_commit / bw_ingest_device
 *       one epoch's items entering the operator: `extract_key`
 *       src/operators.rs:370-416, `routed_exchange` src/timely.rs:809-815,
 *       `InBuffer::extend` src/timely.rs:48-92, then the per-key
 *       `on_batch` loop src/operators.rs:755-806 running
 *       `_WindowLogic.on_batch` windowing.py:1115-1133.
 *   bw_advance
 *       what the operator gives downstream for the activations since the last
 *       call: src/operators.rs:791-794 + `window()`'s three unwrap passes
 *       windowing.py:1321-1338 (down = closed windows, late, meta).
 *   bw_eof
 *       src/operators.rs:862-894 (`on_eof` for every live key, ascending key
 *       order) -> windowing.py:1144-1151.
 *
 * Conventions (SURVEY.md section 8b): no call throws or unwinds; every call
 * returns a bw_status (0 = OK) and leaves a message for bw_last_error().  The
 * library owns all device memory, pinned buffers and communicators; the caller
 * owns only opaque handles.  Handles are not thread-safe; distinct bw_ctx are
 * independent.  No torch / Python types appear anywhere in this file.
 *
 * Times are int64 microseconds since the Unix epoch (the integer form of the
 * reference's aware `datetime`s; UTC_MIN/UTC_MAX as windowing.py:58-62).
 * Keys are uint64; the canonical mapping to the reference's `str` keys
 * (src/operators.rs:401-405) is the decimal string of the integer.
 */
#ifndef BWGPU_H_
#define BWGPU_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BW_ABI_VERSION 1

typedef int32_t bw_status;
enum {
  BW_OK = 0,
  BW_ERR_CUDA = 1,      /* a CUDA runtime call failed */
  BW_ERR_NCCL = 2,      /* an NCCL call failed */
  BW_ERR_CAPACITY = 3,  /* key table / pane pool / emit buffer exhausted */
  BW_ERR_SPEC = 4,      /* invalid bw_fold_spec or argument */
  BW_ERR_STATE = 5,     /* call sequence error (e.g. commit after eof) */
  BW_ERR_RANGE = 6,     /* a timestamp / window id left the representable range */
  BW_ERR_NOMEM = 7
};

#define BW_UTC_MIN_US (-62135596800000000LL)
#define BW_UTC_MAX_US (253402300799999999LL)
/* wait_us value meaning "the watermark never advances on data":
 * EventClock(wait_for_system_duration=timedelta.max), cf.
 * pytests/operators/windowing/test_collect_window.py:33 */
#define BW_WAIT_FOREVER INT64_MAX

typedef enum {
  BW_RED_COUNT = 0, /* count_window: windowing.py:1679-1689 */
  BW_RED_SUM = 1,   /* reduce_window(operator.add): windowing.py:2268-2285 */
  BW_RED_MIN = 2,   /* min_window: windowing.py:2236 */
  BW_RED_MAX = 3,   /* max_window: windowing.py:2189 */
  BW_RED_MEAN = 4   /* fold_window with a (sum, count) accumulator */
} bw_reduction;

typedef enum { BW_VAL_U64 = 0, BW_VAL_I64 = 1, BW_VAL_F32 = 2, BW_VAL_F64 = 3 } bw_val_dtype;

typedef enum {
  BW_TS_COLUMN = 0,     /* ts_us column supplied with every batch */
  BW_TS_FROM_VALUE = 1, /* ts_us = align_to_us + (int64)val: "the value is the
                           event time", examples/benchmark_windowing.py:16-21 */
  BW_TS_NONE = 2        /* no event time: one accumulator per key, emitted by
                           bw_eof in key order as window 0 -- the `*_final`
                           operators (`_FoldFinalLogic`, operators/__init__.py:
                           1923-1950; `reduce_final` :2783-2857, `count_final`
                           :1221-1272, `max_final`/`min_final` :2624-2742).
                           Requires wait_us == BW_WAIT_FOREVER; no ts_us column */
} bw_ts_source;

typedef enum {
  BW_ORDER_REFERENCE = 0, /* rows in the reference's downstream order: per
                             activation, ascending key *string*
                             (src/operators.rs:758-767), then window
                             first-opened order (windowing.py:645-654) */
  BW_ORDER_NONE = 1       /* unordered within an activation (fastest) */
} bw_emit_order;

typedef enum {
  BW_XCHG_P2P = 0, /* partition kernel stores straight into the owning rank's
                      receive buffers over NVLink (CUDA IPC peer mappings) */
  BW_XCHG_NCCL = 1 /* partition into local send buffers, grouped
                      ncclSend/ncclRecv (the baseline transport) */
} bw_exchange;

typedef struct bw_fold_spec {
  uint32_t struct_size; /* sizeof(bw_fold_spec), for ABI growth */
  int32_t reduction;    /* bw_reduction */
  int32_t val_dtype;    /* bw_val_dtype */
  int32_t ts_source;    /* bw_ts_source */
  int64_t length_us;    /* window length  (SlidingWindower.length) */
  int64_t offset_us;    /* window offset; == length_us for tumbling */
  int64_t align_to_us;  /* SlidingWindower.align_to */
  int64_t wait_us;      /* EventClock.wait_for_system_duration, or BW_WAIT_FOREVER */
  int32_t ordered;      /* window(ordered=...) windowing.py:1262 */
  int32_t emit_order;   /* bw_emit_order */
  int32_t exchange;     /* bw_exchange (ignored when world == 1) */
  int32_t ring_slots;   /* pinned ingest slots handed out by bw_ingest_acquire (0 -> 3) */
  uint64_t capacity_hint;  /* expected number of live keys on this rank */
  uint64_t max_batch_rows; /* largest batch a rank will commit / receive */
  uint64_t max_emit_rows;  /* closed-window rows retained between bw_advance calls */
  uint64_t max_late_rows;  /* late rows retained between bw_advance calls */
} bw_fold_spec;

typedef struct bw_ctx bw_ctx;
typedef struct bw_fold bw_fold;

/* A borrowed slot of the pinned ingest ring (valid until the matching commit). */
typedef struct bw_batch {
  uint64_t* keys;  /* [capacity] */
  void* vals;      /* [capacity] of val_dtype (counts carry it only into the late stream) */
  int64_t* ts_us;  /* [capacity]; NULL when ts_source == BW_TS_FROM_VALUE */
  uint64_t capacity;
  uint32_t slot;
  uint32_t reserved;
} bw_batch;

/* Rows handed downstream; host pointers into pinned memory owned by the
 * library, valid until the next bw_advance / bw_eof / bw_fold_destroy. */
typedef struct bw_emit {
  /* `down` + `meta` streams: one row per closed window */
  uint64_t n_closed;
  const uint64_t* closed_key;
  const int64_t* closed_window_id;
  const uint64_t* closed_acc;   /* u64 / i64 / f64 bits (f64 for float sums, MEAN sum) */
  const uint64_t* closed_count; /* number of folded values (MEAN divisor) */
  const uint64_t* closed_epoch; /* epoch of the activation that closed it */
  /* `late` stream: one row per (late item, window it would have been in) */
  uint64_t n_late;
  const uint64_t* late_key;
  const int64_t* late_window_id;
  const uint64_t* late_val; /* value bits */
  const int64_t* late_ts_us;
  const uint64_t* late_epoch;
} bw_emit;

typedef struct bw_stats {
  uint64_t kernel_launches; /* kernels of this library launched so far */
  uint64_t rows_ingested;
  uint64_t rows_received;   /* after the exchange (== ingested when world == 1) */
  uint64_t slow_batches;    /* batches that took the exact out-of-order path */
  uint64_t live_keys;
  uint64_t table_capacity;
  uint64_t pane_nodes_used;
  float last_fold_ms;       /* CUDA-event time of the most recent fold kernel */
  float sum_fold_ms;        /* sum over the TIMED fold launches since bw_fold_create / reset (see timed_folds) */
  uint64_t fold_launches;
  uint64_t fold_rows;
  uint64_t combined_folds;  /* activations folded by the streaming path: bucket scatter + shared-memory segment fold */
  float sum_scatter_ms;     /* CUDA-event time of the k_scatter launches of those activations */
  float sum_verdict_ms;     /* ... and of their k_verdict launches (one each) */
  uint64_t scatter_launches;
  uint64_t split_batches;   /* not-clean activations whose late rows were found without the sort (streaming fold for the rest) */
  uint64_t timed_folds;     /* fold launches behind sum_fold_ms / fold_rows: every BW_TIMER_STRIDE-th activation (default 4) is
                             * timed -- an event record with timing drains the stream for a few microseconds */
  uint64_t scatter_spill_rows; /* rows the bucket scatter put in the spill list (a lane was full), summed over activations */
} bw_stats;

/* ---- context ---------------------------------------------------------- */

/* Fill `out128` with an NCCL unique id (rank 0 calls this and ships the bytes
 * to the other ranks by any means; 128 bytes). */
bw_status bw_nccl_unique_id(void* out128);

/* `nccl_unique_id` may be NULL iff world == 1. */
bw_status bw_ctx_create(int device, int rank, int world, const void* nccl_unique_id, bw_ctx** out);
void bw_ctx_destroy(bw_ctx* ctx);
/* Test harness for boxes with one GPU: a world whose ranks are THREADS of one process on one device.  The collectives
 * become host rendezvous, peer memory plain pointers; kernels, arguments and results are those of the NCCL / CUDA-IPC
 * world, so the whole multi-rank path (bw_route, partition, exchange, combine / merge -- src/timely.rs:455-569, 809-815)
 * can be checked without a second GPU.  Only the P2P exchange; every rank thread makes the same sequence of calls. */
typedef struct bw_loopback bw_loopback;
bw_status bw_loopback_create(int world, bw_loopback** out);
void bw_loopback_destroy(bw_loopback* world);
bw_status bw_ctx_create_loopback(int device, int rank, bw_loopback* world, bw_ctx** out);
const char* bw_last_error(const bw_ctx* ctx);
/* Message of the last failure that had no ctx (bw_ctx_create itself). */
const char* bw_last_global_error(void);
uint32_t bw_abi_version(void);

/* Owning rank of a key: (mix64(key) >> 32) * world >> 32. */
uint32_t bw_route(uint64_t key, uint32_t world);

/* ---- fold -------------------------------------------------------------- */

bw_status bw_fold_create(bw_ctx* ctx, const bw_fold_spec* spec, bw_fold** out);
void bw_fold_destroy(bw_fold* fold);

/* Borrow a pinned host slot able to hold `max_rows` rows. */
bw_status bw_ingest_acquire(bw_fold* fold, uint64_t max_rows, bw_batch* out);

/* Submit `rows` rows of a slot as one activation at `epoch`: async H2D, then
 * (world > 1) partition + exchange, then the fold.  Returns without waiting
 * for the device.  Collective when world > 1: every rank commits the same
 * sequence of epochs (a rank with no data commits rows == 0). */
bw_status bw_ingest_commit(bw_fold* fold, const bw_batch* batch, uint64_t rows, uint64_t epoch);

/* Same as acquire+commit for columns already resident in device memory.
 * Lifetime: with world == 1 the fold reads the columns in place, so they must
 * stay valid and unchanged until bw_fold_sync / bw_advance / bw_eof returns
 * (or be overwritten only by work enqueued on bw_fold_stream, which is ordered
 * behind the fold); with world > 1 they are consumed by the exchange before
 * the call returns.  The columns must be completely written before the call:
 * the lateness pass (and, when world > 1, the exchange) runs on its own stream
 * so that it overlaps the previous activation's fold, and takes no ordering
 * from the fold's stream (columns produced by bw_gen_c1 on this fold are
 * ordered by the library itself). */
bw_status bw_ingest_device(bw_fold* fold, const uint64_t* d_keys, const void* d_vals,
                           const int64_t* d_ts_us, uint64_t rows, uint64_t epoch);

/* System time of the activations committed from now on (`now_getter()` sampled by `before_batch`, windowing.py:250-261;
 * microseconds since the Unix epoch, never goes backwards).  The EventClock's watermark of a key is
 *   max_j(ts_j - wait - now_j) + now      (windowing.py:263-287: watermark_base + (now - system_time_of_max_event))
 * so an item is late, and a window closes, against a watermark that also drifts forward with the system clock.
 * Never called: the frozen clock (now == 0 throughout), the watermark is max(ts) - wait.  One rank only. */
bw_status bw_fold_set_system_now(bw_fold* fold, int64_t system_now_us);

/* Wait for every committed activation and return what they emitted.
 * `system_now_us` > 0 additionally runs the reference's notify phase (src/operators.rs:808-858) at that system time:
 * every key whose earliest open window's close time has been reached by the system clock (`notify_at`,
 * windowing.py:656-659, 1146-1173) closes what its watermark now allows (`on_notify`, windowing.py:1137-1144) -- an
 * idle key's windows no longer wait for EOF.  0: data-driven only (frozen clock).  `closed_epoch` is accepted and
 * unused (epochs are closed by the order of the commits). */
bw_status bw_advance(bw_fold* fold, uint64_t closed_epoch, int64_t system_now_us, bw_emit* out);

/* End of input: watermark := UTC_MAX, every open window closes (ascending key
 * order), all state is dropped.  Collective when world > 1. */
bw_status bw_eof(bw_fold* fold, bw_emit* out);

/* ---- snapshot / restore (SURVEY 8f row 3) ------------------------------
 * One row per live (key, pane): what `_WindowLogic.snapshot` captures per key
 * (`_WindowSnapshot`, pysrc/bytewax/operators/windowing.py:1032-1037,
 * 1182-1190: clock state, open windows, accumulators) in columnar form, for a
 * recovery store to persist (src/operators.rs:931-1003 writes one snapshot per
 * awoken key per epoch; src/recovery.rs:1520-1614 reads them back). */
typedef struct bw_snapshot {
  uint64_t n;                  /* rows */
  const uint64_t* key;
  const int64_t* pane_id;      /* window id for tumbling windows; pane (gcd(length, offset)) id for sliding */
  const uint64_t* acc;         /* accumulator bits, as bw_emit.closed_acc before the float decoding of min/max */
  const uint64_t* count;       /* folded values (MEAN divisor) */
  const uint64_t* open_seq;    /* first-open order of the pane: activation << 32 | arrival index */
  const int64_t* max_ts_us;    /* per key (repeated on each of its rows): the event clock's state */
  const int64_t* closed_upto;  /* sliding: last window id already emitted for the key, INT64_MIN if none */
  uint64_t batch_no;           /* activations folded so far (keeps open_seq ordered across a restore) */
  int64_t gmax_ts_us;          /* running max event time over everything ingested (lateness verdict) */
  uint64_t last_epoch;
} bw_snapshot;

/* Dump the state after the last bw_advance.  Host pointers into pinned memory
 * owned by the library, valid until the next bw_snapshot_take / destroy. */
bw_status bw_snapshot_take(bw_fold* fold, bw_snapshot* out);
/* Load a dump into a freshly created fold with the same window spec (capacity
 * and world size may differ: rows are re-inserted by key; with world > 1 every
 * rank passes the full row set and keeps the keys it owns, the reference's
 * rescale on resume, src/recovery.rs:1701-1781). */
bw_status bw_snapshot_load(bw_fold* fold, const bw_snapshot* in);

/* Window bounds for the `meta` stream: WindowMetadata(open_time, close_time),
 * windowing.py:620-623. */
void bw_window_bounds(const bw_fold_spec* spec, int64_t window_id, int64_t* open_us, int64_t* close_us);

bw_status bw_fold_stats(bw_fold* fold, bw_stats* out);
/* Zero the timing counters of bw_stats (not the state). */
bw_status bw_fold_reset_timers(bw_fold* fold);
/* Block until all work submitted on this fold's streams has finished. */
bw_status bw_fold_sync(bw_fold* fold);
/* CUDA-event stopwatch on the launching stream (bench): begin records an event
 * on the fold's compute stream; end records a second one, waits for it and
 * returns the elapsed device time in milliseconds. */
bw_status bw_fold_time_begin(bw_fold* fold);
bw_status bw_fold_time_end(bw_fold* fold, float* ms);
/* cudaStream_t (as void*) that the fold / partition kernels are launched on. */
void* bw_fold_stream(bw_fold* fold);

/* Fill device columns with SURVEY.md section 8(d) config C1 rows
 * [start, start+rows): key = splitmix64(0x5EED ^ i) mod n_keys, val = i.
 * Test/bench input generation only; launched on the fold's stream. */
bw_status bw_gen_c1(bw_fold* fold, uint64_t* d_keys, uint64_t* d_vals, uint64_t start, uint64_t rows,
                    uint64_t n_keys);

/* ---- keyed steps that are not window folds (BASELINE configs C2 and C4) ---------------- */

/* `stateful_map` with the rolling z-score mapper of examples/anomaly_detector.py:16-48, run by
 * `_StatefulLogic.on_batch` / `_StatefulFlatMapLogic.on_item`
 * (pysrc/bytewax/operators/__init__.py:1024-1042, 2860-2890) behind src/operators.rs:755-806:
 * per key, in arrival order: flag = |v - mu| / sigma > threshold on the statistics BEFORE the
 * push (false while mu or sigma is None or 0.0), then push v into the last-`window` ring and
 * recompute mu = sum/len, sigma = sqrt(sum((x - mu)^2)/len), both newest -> oldest. */
typedef struct bw_smap bw_smap;
typedef struct bw_smap_spec {
  uint32_t struct_size;
  int32_t window;      /* ring length, 1..32 (the example uses 10) */
  int32_t val_dtype;   /* BW_VAL_F32 or BW_VAL_F64 */
  int32_t reserved;
  double threshold;    /* the example uses 2.0 */
  uint64_t capacity_hint;
  uint64_t max_batch_rows;
} bw_smap_spec;
bw_status bw_smap_create(bw_ctx* ctx, const bw_smap_spec* spec, bw_smap** out);
void bw_smap_destroy(bw_smap* m);
/* One activation from HOST columns; outputs are aligned with the input rows. Blocking. */
bw_status bw_smap_apply(bw_smap* m, const uint64_t* keys, const void* vals, uint64_t rows, double* out_mu,
                        double* out_sigma, uint8_t* out_flag);
/* Same with DEVICE columns in and out (returns after enqueueing; bw_smap_sync to wait). */
bw_status bw_smap_apply_device(bw_smap* m, const uint64_t* d_keys, const void* d_vals, uint64_t rows, double* d_mu,
                               double* d_sigma, uint8_t* d_flag);
bw_status bw_smap_sync(bw_smap* m);

/* Two-sided keyed join: `_JoinLogic.on_item` / `on_eof` (operators/__init__.py:2157-2190) over the
 * side-labelled merged stream of `_join_label_merge` (:2193-2204); insert modes first / last,
 * emit modes complete / final / running (`product` keeps lists per side: host path only). */
typedef enum { BW_JOIN_INSERT_FIRST = 0, BW_JOIN_INSERT_LAST = 1 } bw_join_insert;
typedef enum { BW_JOIN_EMIT_COMPLETE = 0, BW_JOIN_EMIT_FINAL = 1, BW_JOIN_EMIT_RUNNING = 2 } bw_join_emit_mode;
typedef struct bw_join bw_join;
typedef struct bw_join_spec {
  uint32_t struct_size;
  int32_t insert_mode;
  int32_t emit_mode;
  int32_t reserved;
  uint64_t capacity_hint;
  uint64_t max_batch_rows;
  uint64_t max_emit_rows;
} bw_join_spec;
typedef struct bw_join_rows {
  uint64_t n;
  const uint64_t* key;
  const uint64_t* left;   /* valid where mask bit 0 is set (else the reference emits None) */
  const uint64_t* right;  /* valid where mask bit 1 is set */
  const uint64_t* mask;
  const uint64_t* epoch;
} bw_join_rows;
bw_status bw_join_create(bw_ctx* ctx, const bw_join_spec* spec, bw_join** out);
void bw_join_destroy(bw_join* j);
/* One activation: items of both sides in arrival order, side[i] in {0 = left, 1 = right}; host columns. */
bw_status bw_join_apply(bw_join* j, const uint64_t* keys, const uint8_t* side, const uint64_t* vals, uint64_t rows,
                        uint64_t epoch);
/* Rows emitted since the last call, reference order: per activation ascending key string, then item order. */
bw_status bw_join_advance(bw_join* j, bw_join_rows* out);
bw_status bw_join_eof(bw_join* j, bw_join_rows* out);

/* Session-window fold (K7): `_WindowLogic` (unordered) over `_SessionWindowerLogic` with a numeric fold,
 * pysrc/bytewax/operators/windowing.py:1046-1190 and :671-810, built by `SessionWindower` :928-950.  Per key, in
 * arrival order: the EventClock's late test (:263-287, :1125-1127; a late item gives one row with window id
 * LATE_SESSION_ID = -1, :671, :764-766); `open_for` (:731-762): the FIRST live session by id that contains the
 * timestamp, or whose open is 0 < open - ts <= gap ahead (open := ts), or whose close is 0 < ts - close <= gap
 * behind (close := ts), else a new session with id max_key + 1 (max_key starts at -1 and never resets: session
 * state is never discarded, :798-806); after an extension `_session_find_merges` (:688-715) merges, in open order,
 * every session that opens within gap of the running survivor's close into the EARLIEST-OPENED one, which gains the
 * merged id (direct merges only).  Then the activation's inserts are folded (:1064-1077) into the accumulator of the
 * id `open_for` returned, then the merge queue in discovery order (`into = merger(into, orig)`, :1079-1085), then
 * `close_for` (:774-788): sessions with close < watermark - gap (UTC_MIN if that is below it), in id order.
 * Accumulators: count_window :1679-1689; reduce_window(operator.add) :2268-2285 (i64 sums wrap past 2^63);
 * max_window / min_window :2189 / :2236 with `by` = identity (the accumulator is replaced only if the new value is
 * strictly greater / less, so signed zeros and NaN come out exactly as in Python).  One GPU only. */
typedef struct bw_session bw_session;
typedef struct bw_session_spec {
  uint32_t struct_size;
  int32_t reduction;            /* BW_RED_COUNT / SUM / MIN / MAX */
  int32_t val_dtype;            /* BW_VAL_I64 or BW_VAL_F64 (values are ignored by count) */
  int32_t max_sessions_per_key; /* 1..64: sessions a key holds during an activation (live ones, plus those merged away
                                   in it, which keep their accumulator until the activation's merge pass), and also the
                                   merged ids its live sessions hold */
  int64_t gap_us;               /* SessionWindower.gap, >= 0 (windowing.py:938-943) */
  int64_t wait_us;              /* EventClock.wait_for_system_duration, or BW_WAIT_FOREVER */
  uint64_t capacity_hint;       /* keys ever seen: session state is never freed (windowing.py:798-806) */
  uint64_t max_batch_rows;
  uint64_t max_emit_rows;       /* closed sessions, and their merged ids, retained between bw_session_advance calls */
  uint64_t max_late_rows;       /* late rows retained between bw_session_advance calls */
} bw_session_spec;
/* Rows handed downstream since the last advance / eof, in the reference's order: per call (activation, notify phase
 * or EOF), ascending key string (src/operators.rs:758-767, :862-894); within a key late rows in arrival order and
 * closed sessions in id order.  Host pointers into memory owned by the library, valid until the next advance / eof /
 * destroy. */
typedef struct bw_session_rows {
  /* `down` + `meta` streams: one row per closed session, WindowMetadata(open, close, merged_ids) (:1087-1093) */
  uint64_t n_closed;
  const uint64_t* closed_key;
  const int64_t* closed_window_id;
  const uint64_t* closed_acc;     /* count: u64; sum / min / max: i64 or f64 bits */
  const int64_t* closed_open_us;
  const int64_t* closed_close_us;
  const uint64_t* closed_epoch;   /* the epoch of the activation, or of the last one before a notify / EOF */
  const uint64_t* merged_off;     /* [n_closed + 1]: row i merged ids are merged_ids[merged_off[i] .. merged_off[i+1]) */
  const int64_t* merged_ids;      /* ascending per row */
  /* `late` stream: one row per late item; (activation, row) name the input row (activations counted from 0) */
  uint64_t n_late;
  const uint64_t* late_key;
  const uint64_t* late_epoch;
  const uint64_t* late_activation;
  const uint64_t* late_row;
} bw_session_rows;
bw_status bw_session_create(bw_ctx* ctx, const bw_session_spec* spec, bw_session** out);
void bw_session_destroy(bw_session* s);
/* One activation from HOST columns (vals may be NULL for count); blocks.  `system_now_us` is `now_getter()` for this
 * activation (windowing.py:250-261; it must not go backwards; 0 throughout = a frozen clock).  The key's watermark is
 * then max_j(ts_j - wait - now_j) + now, as bw_fold_set_system_now describes. */
bw_status bw_session_apply(bw_session* s, const uint64_t* keys, const void* vals, const int64_t* ts_us, uint64_t rows,
                           uint64_t epoch, int64_t system_now_us);
/* Same with DEVICE columns; returns once the work is enqueued (the columns must stay valid until the next call). */
bw_status bw_session_apply_device(bw_session* s, const uint64_t* d_keys, const void* d_vals, const int64_t* d_ts_us,
                                  uint64_t rows, uint64_t epoch, int64_t system_now_us);
/* Rows since the last call.  `system_now_us` > 0 first runs the notify phase at that system time
 * (src/operators.rs:808-858, windowing.py:1135-1142, 1153-1180 with an identity `to_system_utc`): every key with a
 * live session whose earliest close + gap has been reached closes what its watermark at that time allows. */
bw_status bw_session_advance(bw_session* s, int64_t system_now_us, bw_session_rows* out);
/* End of input: watermark := UTC_MAX (:300-302), so sessions with close >= UTC_MAX - gap stay open. */
bw_status bw_session_eof(bw_session* s, bw_session_rows* out);

/* Windowed join (K8): `join_window` (pysrc/bytewax/operators/windowing.py:2056-2140) with insert modes first / last,
 * i.e. `_WindowLogic` (:1046-1190) over `_SlidingWindowerLogic` (:603-668; tumbling == offset equal to length,
 * :921-926) with `_JoinWindowLogic` (:1849-1902) per window.  Values travel as u64 handles; the objects stay with the
 * caller.  Per key, per call, in order: the EventClock's late test per item (:263-287; a late item gives one row per id
 * of `intersects(ts)`, ascending, :611-618, :636-637, :1125-1127, and is not queued); `_flush_queue` (:1095-1108) at the
 * watermark after the key's last item: unordered, every queued entry in arrival order; ordered, the entries with
 * ts <= watermark, stably sorted by ts, the rest kept queued in their order across calls; each due entry goes to every
 * window of `open_for(ts)` in ascending id (:626-633, :1064-1077; a window is opened on its first value), where "first"
 * sets its side only if unset, "last" always (:1866-1876, `_JoinState` operators/__init__.py:2076-2120), "complete" emits
 * the tuple and clears the state once every side is set, "running" emits the tuple after every value; then
 * `_handle_closed` (:1087-1093): windows with close <= watermark in first-opened order, each giving the `final` tuple
 * (emit mode final) and then its metadata row.  A key with no open window and an empty queue is discarded, clock state
 * included (:1110-1113, src/operators.rs:796-799).  One GPU only. */
typedef struct bw_jwin bw_jwin;
typedef struct bw_jwin_spec {
  uint32_t struct_size;
  int32_t insert_mode;          /* BW_JOIN_INSERT_FIRST / LAST (product keeps lists per side: host engine) */
  int32_t emit_mode;            /* BW_JOIN_EMIT_COMPLETE / FINAL / RUNNING */
  int32_t ordered;              /* 1: play values in timestamp order once the watermark passes them (the default) */
  int32_t sides;                /* 1..4 joined streams */
  int32_t max_windows_per_key;  /* 1..64 open windows per key */
  int64_t length_us;            /* window length, > 0 */
  int64_t offset_us;            /* 0 < offset <= length (TumblingWindower: == length) */
  int64_t align_us;             /* align_to */
  int64_t wait_us;              /* EventClock.wait_for_system_duration, or BW_WAIT_FOREVER */
  uint64_t capacity_hint;       /* live keys; a key's slot is kept once seen */
  uint64_t max_queued_rows;     /* ordered mode: queued entries over ALL keys (with a long wait one key may hold most) */
  uint64_t max_batch_rows;
  uint64_t max_emit_rows;       /* down rows, and meta rows, retained between bw_jwin_advance calls */
  uint64_t max_late_rows;       /* late rows retained between bw_jwin_advance calls */
} bw_jwin_spec;
/* Rows handed downstream since the last advance / eof, in the reference's order: per call (activation, notify phase
 * or EOF), ascending key string (src/operators.rs:758-767, :862-894); within a key `down` rows in play order with the
 * close-time (`final`) rows after them, `meta` rows in first-opened order, `late` rows in arrival order (one per window
 * id, ascending).  Host pointers into memory owned by the library, valid until the next advance / eof / destroy. */
typedef struct bw_jwin_rows {
  uint64_t n_down;
  const uint64_t* down_key;
  const int64_t* down_window_id;
  const uint64_t* down_handle[4]; /* [side][row]: valid where bit `side` of down_mask is set (else the reference emits None) */
  const uint64_t* down_mask;
  const uint64_t* down_epoch;
  uint64_t n_meta;                /* closed windows: WindowMetadata(align + id * offset, + length) */
  const uint64_t* meta_key;
  const int64_t* meta_window_id;
  const uint64_t* meta_epoch;
  uint64_t n_late;
  const uint64_t* late_key;
  const int64_t* late_window_id;
  const uint64_t* late_epoch;
  const uint64_t* late_activation; /* (activation, row) name the input row (activations counted from 0) */
  const uint64_t* late_row;
  /* handles no window and no queue entry holds any more; each handle passed to apply is listed exactly once, in the
   * rows of the call that let go of it (late items and values never stored: the call that received them) */
  uint64_t n_released;           /* (the device buffer behind it grows with the handles held, never with the table size) */
  const uint64_t* released;
} bw_jwin_rows;
bw_status bw_jwin_create(bw_ctx* ctx, const bw_jwin_spec* spec, bw_jwin** out);
void bw_jwin_destroy(bw_jwin* j);
/* One activation from HOST columns (keys, side 0..sides-1, handle, ts); blocks.  `system_now_us` is `now_getter()`
 * for this activation (windowing.py:250-261; it must not go backwards; 0 throughout = a frozen clock). */
bw_status bw_jwin_apply(bw_jwin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us,
                        uint64_t rows, uint64_t epoch, int64_t system_now_us);
/* Same with DEVICE columns; returns once the work is enqueued (the columns must stay valid until the next call).  A side
 * value >= sides is not played: the next call returns BW_ERR_SPEC and the join refuses further calls. */
bw_status bw_jwin_apply_device(bw_jwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles,
                               const int64_t* d_ts_us, uint64_t rows, uint64_t epoch, int64_t system_now_us);
/* Rows since the last call.  `system_now_us` > 0 first runs the notify phase at that system time
 * (src/operators.rs:808-858, windowing.py:1135-1142, 1153-1180 with an identity `to_system_utc`): every key whose
 * earliest window close -- or, ordered, the ts of its FIRST queued entry -- has been reached flushes at its watermark. */
bw_status bw_jwin_advance(bw_jwin* j, int64_t system_now_us, bw_jwin_rows* out);
/* End of input: every key flushes at watermark UTC_MAX (:1144-1151). */
bw_status bw_jwin_eof(bw_jwin* j, bw_jwin_rows* out);

/* Windowed collect (K9): `collect_window` (pysrc/bytewax/operators/windowing.py:1436-1576) into list / set / dict,
 * i.e. `_WindowLogic` (:1046-1190) over `_SlidingWindowerLogic` (:603-668; tumbling == offset equal to length,
 * :921-926) with `_FoldWindowLogic` per window and the collect callbacks (:1356-1384), whose state is the window's
 * values in play order.  Values travel as u64 handles (any u64: none is reserved); the objects stay with the caller,
 * which builds each container from the window's handles -- `into()`, then `append` / `add` / `d[k] = v` per handle in
 * order, exactly the reference's folder calls.  Per key, per call, in order: the EventClock's late test per item
 * (:263-287; a late item gives one row per id of `intersects(ts)`, ascending, :611-618, :636-637, :1125-1127, and is not
 * queued); `_flush_queue` (:1095-1108) at the watermark after the key's last item: unordered, every queued entry in
 * arrival order; ordered, the entries with ts <= watermark, stably sorted by ts, the rest kept queued in their order
 * across calls; each due value joins every window of `open_for(ts)` in ascending id (:626-633, :1064-1077; a window is
 * opened on its first value); then `_handle_closed` (:1087-1093): windows with close <= watermark in first-opened order,
 * each giving its list and then its metadata row.  A key with no open window and an empty queue is discarded, clock
 * state included (:1110-1113, src/operators.rs:796-799).  One GPU only. */
typedef struct bw_collect bw_collect;
typedef struct bw_collect_spec {
  uint32_t struct_size;
  int32_t ordered;              /* 1: play values in timestamp order once the watermark passes them (the default) */
  int32_t max_windows_per_key;  /* 1..64 open windows per key */
  int32_t pad;
  int64_t length_us;            /* window length, > 0 */
  int64_t offset_us;            /* 0 < offset <= length (TumblingWindower: == length) */
  int64_t align_us;             /* align_to */
  int64_t wait_us;              /* EventClock.wait_for_system_duration, or BW_WAIT_FOREVER */
  uint64_t capacity_hint;       /* live keys; a key's slot is kept once seen */
  uint64_t max_queued_rows;     /* ordered mode: queued entries over ALL keys */
  uint64_t max_batch_rows;
  uint64_t max_emit_rows;       /* closed windows retained between bw_collect_advance calls */
  uint64_t max_late_rows;       /* late rows retained between bw_collect_advance calls */
} bw_collect_spec;
/* Rows handed downstream since the last advance / eof, in the reference's order: per call (activation, notify phase
 * or EOF), ascending key string (src/operators.rs:758-767, :862-894); within a key `down` rows in first-opened order,
 * `late` rows in arrival order (one per window id, ascending).  Each down row is one closed window: its `E` row is the
 * list handle[down_offset[i] .. down_offset[i + 1]) (play order), and its `M` row, which follows it, is
 * WindowMetadata(align + id * offset, + length) -- so no separate meta columns.  Host pointers into memory owned by the
 * library, valid until the next advance / eof / destroy. */
typedef struct bw_collect_rows {
  uint64_t n_down;
  const uint64_t* down_key;
  const int64_t* down_window_id;
  const uint64_t* down_epoch;
  const uint64_t* down_offset;     /* n_down + 1 entries */
  const uint64_t* handle;          /* down_offset[n_down] entries */
  uint64_t n_late;
  const uint64_t* late_key;
  const int64_t* late_window_id;
  const uint64_t* late_epoch;
  const uint64_t* late_activation; /* (activation, row) name the input row (activations counted from 0) */
  const uint64_t* late_row;
  /* handles no window and no queue entry holds any more: each handle passed to apply is listed exactly once, in the
   * rows of the call that closes the last window holding it (its highest id of `open_for(ts)`: a key's windows close
   * in id order), a late item's in the call that received it */
  uint64_t n_released;
  const uint64_t* released;
} bw_collect_rows;
bw_status bw_collect_create(bw_ctx* ctx, const bw_collect_spec* spec, bw_collect** out);
void bw_collect_destroy(bw_collect* c);
/* One activation from HOST columns (keys, handle, ts); blocks.  `system_now_us` is `now_getter()` for this activation
 * (windowing.py:250-261; it must not go backwards; 0 throughout = a frozen clock).  The entry store, the staging and
 * output buffers and the release buffer grow before each call to what it can add, so no call fails for lack of room
 * there; a full key table, window list, queue, late buffer or closed-window buffer returns BW_ERR_CAPACITY (reason in
 * bw_last_error) and the collect refuses further calls. */
bw_status bw_collect_apply(bw_collect* c, const uint64_t* keys, const uint64_t* handles, const int64_t* ts_us, uint64_t rows,
                           uint64_t epoch, int64_t system_now_us);
/* Same with DEVICE columns; returns once the work is enqueued (the columns must stay valid until the next call). */
bw_status bw_collect_apply_device(bw_collect* c, const uint64_t* d_keys, const uint64_t* d_handles, const int64_t* d_ts_us,
                                  uint64_t rows, uint64_t epoch, int64_t system_now_us);
/* Rows since the last call.  `system_now_us` > 0 first runs the notify phase at that system time
 * (src/operators.rs:808-858, windowing.py:1135-1142, 1153-1180 with an identity `to_system_utc`): every key whose
 * earliest window close -- or, ordered, the ts of its FIRST queued entry -- has been reached flushes at its watermark. */
bw_status bw_collect_advance(bw_collect* c, int64_t system_now_us, bw_collect_rows* out);
/* End of input: every key flushes at watermark UTC_MAX (:1144-1151). */
bw_status bw_collect_eof(bw_collect* c, bw_collect_rows* out);

/* Windowed join over session windows (K10): `join_window` (pysrc/bytewax/operators/windowing.py:2056-2140) with insert
 * modes first / last over `SessionWindower` (:928-950), i.e. `_WindowLogic` (:1046-1190) over `_SessionWindowerLogic`
 * (:671-810) with `_JoinWindowLogic` (:1849-1902) per session.  Values travel as u64 handles; the objects stay with the
 * caller.  Per key, per call, in order: the EventClock's late test per item (:263-287; a late item gives one row, window
 * LATE_SESSION_ID = -1, :671, :764-766, and is not queued); `_flush_queue` (:1095-1108) at the watermark after the key's
 * last item (unordered: every queued entry in arrival order; ordered: the entries with ts <= watermark, stably sorted by
 * ts, the rest kept queued across calls); per due value `open_for` (:731-762: the FIRST live session by id that contains
 * ts or lies within gap of it, extended, then `_session_find_merges` :688-715; else a new session, id max_key + 1) and
 * `on_value` on the session it returned, even one a merge just took away (:1064-1077, :1866-1876); then the merge queue
 * in discovery order (:1079-1085) with `on_merge` (:1879-1891): "first" takes the merged-away session's value on every
 * side it set, "last" keeps the survivor's on every side the survivor set; then "complete" emits under the survivor's id
 * and clears once every side is set, "running" emits; then `close_for` (:774-788): sessions with close < watermark - gap
 * (UTC_MIN if that is below it) in id order, each giving the `final` tuple (emit mode final) and its metadata row.
 * Session state is never discarded (:798-806): a key's clock and session ids outlive its sessions.  One GPU only. */
typedef struct bw_sjwin bw_sjwin;
typedef struct bw_sjwin_spec {
  uint32_t struct_size;
  int32_t insert_mode;          /* BW_JOIN_INSERT_FIRST / LAST (product keeps lists per side: host engine) */
  int32_t emit_mode;            /* BW_JOIN_EMIT_COMPLETE / FINAL / RUNNING */
  int32_t ordered;              /* 1: play values in timestamp order once the watermark passes them (the default) */
  int32_t sides;                /* 1..4 joined streams */
  int32_t max_sessions_per_key; /* 1..64: sessions a key holds during a call (live ones, plus those merged away in it),
                                   and also the merged ids its live sessions hold */
  int64_t gap_us;               /* SessionWindower.gap, >= 0 (windowing.py:938-943) */
  int64_t wait_us;              /* EventClock.wait_for_system_duration, or BW_WAIT_FOREVER */
  uint64_t capacity_hint;       /* keys ever seen: session state is never freed (windowing.py:798-806) */
  uint64_t max_queued_rows;     /* ordered mode: queued entries over ALL keys */
  uint64_t max_batch_rows;
  uint64_t max_emit_rows;       /* down rows, meta rows, and meta rows' merged ids, retained between bw_sjwin_advance calls */
  uint64_t max_late_rows;       /* late rows retained between bw_sjwin_advance calls */
} bw_sjwin_spec;
/* Rows handed downstream since the last advance / eof, in the reference's order: per call (activation, notify phase
 * or EOF), ascending key string (src/operators.rs:758-767, :862-894); within a key `down` rows of the inserts in play
 * order, then of the merges in merge-queue order (under the survivor's id), then the `final` rows of the closing
 * sessions in id order; `meta` rows in id order; `late` rows in arrival order.  Host pointers into memory owned by the
 * library, valid until the next advance / eof / destroy. */
typedef struct bw_sjwin_rows {
  uint64_t n_down;
  const uint64_t* down_key;
  const int64_t* down_window_id;
  const uint64_t* down_handle[4]; /* [side][row]: valid where bit `side` of down_mask is set (else the reference emits None) */
  const uint64_t* down_mask;
  const uint64_t* down_epoch;
  uint64_t n_meta;                /* closed sessions: WindowMetadata(open, close, merged_ids) */
  const uint64_t* meta_key;
  const int64_t* meta_window_id;
  const int64_t* meta_open_us;
  const int64_t* meta_close_us;
  const uint64_t* meta_epoch;
  const uint64_t* merged_off;     /* [n_meta + 1]: row i merged ids are merged_ids[merged_off[i] .. merged_off[i+1]) */
  const int64_t* merged_ids;      /* ascending per row: the sessions merged directly into it */
  uint64_t n_late;                /* window id LATE_SESSION_ID = -1 */
  const uint64_t* late_key;
  const uint64_t* late_epoch;
  const uint64_t* late_activation; /* (activation, row) name the input row (activations counted from 0) */
  const uint64_t* late_row;
  /* handles no session and no queue entry holds any more; each handle passed to apply is listed exactly once, in the
   * rows of the call that let go of it: a late item's and a "first" value's that found its side set in the call that
   * received it; a value replaced by "last", cleared by "complete" or losing a merge; a session's when it closes */
  uint64_t n_released;           /* (the device buffer behind it grows with the handles held, never with the table size) */
  const uint64_t* released;
} bw_sjwin_rows;
/* windowing.py:2056-2140 (join_window) + :1046-1190 (_WindowLogic) + :671-810 (_SessionWindowerLogic) */
bw_status bw_sjwin_create(bw_ctx* ctx, const bw_sjwin_spec* spec, bw_sjwin** out);
void bw_sjwin_destroy(bw_sjwin* j);
/* One activation from HOST columns (keys, side 0..sides-1, handle, ts); blocks: `_WindowLogic.on_batch`
 * (windowing.py:1115-1133).  `system_now_us` is `now_getter()` for this activation (:250-261; it must not go backwards;
 * 0 throughout = a frozen clock).  A full key table, more than max_sessions_per_key sessions or merged ids, or a full
 * queue, emit or late buffer returns BW_ERR_CAPACITY (reason in bw_last_error) and the join refuses further calls. */
bw_status bw_sjwin_apply(bw_sjwin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us,
                         uint64_t rows, uint64_t epoch, int64_t system_now_us);
/* Same with DEVICE columns; returns once the work is enqueued (the columns must stay valid until the next call).  A side
 * value >= sides is not played: the next call returns BW_ERR_SPEC and the join refuses further calls. */
bw_status bw_sjwin_apply_device(bw_sjwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles,
                                const int64_t* d_ts_us, uint64_t rows, uint64_t epoch, int64_t system_now_us);
/* Rows since the last call.  `system_now_us` > 0 first runs the notify phase at that system time
 * (src/operators.rs:808-858, windowing.py:1135-1142, 1153-1180 with an identity `to_system_utc`): every key whose
 * earliest session close + gap -- or, ordered, the ts of its FIRST queued entry -- has been reached flushes at its
 * watermark. */
bw_status bw_sjwin_advance(bw_sjwin* j, int64_t system_now_us, bw_sjwin_rows* out);
/* End of input: every key flushes at watermark UTC_MAX (:1144-1151), so sessions with close >= UTC_MAX - gap stay open. */
bw_status bw_sjwin_eof(bw_sjwin* j, bw_sjwin_rows* out);

/* ---- plain device-memory helpers (tests / bench / host bindings without torch) ---- */
bw_status bw_dev_alloc(bw_ctx* ctx, uint64_t bytes, void** out);
bw_status bw_dev_free(bw_ctx* ctx, void* ptr);
bw_status bw_host_alloc(bw_ctx* ctx, uint64_t bytes, void** out); /* pinned */
bw_status bw_host_free(bw_ctx* ctx, void* ptr);
/* kind: 0 = host->device, 1 = device->host, 2 = device->device; synchronous */
bw_status bw_memcpy(bw_ctx* ctx, void* dst, const void* src, uint64_t bytes, int kind);
/* Write `bytes` of 0xA5 to a scratch device buffer larger than L2 (bench L2 flush). */
bw_status bw_flush_l2(bw_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* BWGPU_H_ */
