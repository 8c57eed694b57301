// bw_fold.cuh -- K3: window-assign + open-addressed hash-table fold.
//
// Replaces the per-key `on_batch` loop of src/operators.rs:755-806 running
// `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) for
// numeric folds.  One thread per event.
//
// Steady state (key known, event falls in the key's newest pane): ONE 32-byte
// sector read (two LDG.128) and one or two fire-and-forget L2 reductions.  Every
// other case (second probe, new key, second pane, further panes) is pushed to
// a block-local queue and drained by full warps afterwards, so the rare,
// latency-bound paths never hold the fast lanes of a warp hostage.
#pragma once
#include "bw_common.cuh"

// Compile-time specialisation of the fold: the accumulator op, whether the
// watermark is tracked and whether value counts are kept are template
// constants in the hot kernel (one small instruction stream per fold type --
// the generic kernel was 74 KB of SASS and stalled on instruction fetch);
// -1 means "read it from FoldParams at run time" (exact slow path).
template <int OP_, int WM_, int CNT_>
struct FoldCfg {
  static constexpr int kOp = OP_, kWm = WM_, kCnt = CNT_;
  __device__ __forceinline__ static int op(const FoldParams& p) { return OP_ >= 0 ? OP_ : p.op; }
  __device__ __forceinline__ static bool wm(const FoldParams& p) { return WM_ >= 0 ? (WM_ != 0) : (p.track_wm != 0); }
  __device__ __forceinline__ static bool cnt(const FoldParams& p) { return CNT_ >= 0 ? (CNT_ != 0) : (p.need_count != 0); }
};
typedef FoldCfg<-1, -1, -1> FoldCfgRuntime;

// Block-local staging of the rare global appends (dirty-key list, new-key
// count) and of the deferred events.
#define BW_SINK_CAP 1024
#define BW_FOLD_THREADS 256
#ifndef BW_FOLD_UNROLL
#define BW_FOLD_UNROLL 4
#endif
#ifndef BW_FOLD_MINB
#define BW_FOLD_MINB 3
#endif
#define BW_FOLD_WARPS (BW_FOLD_THREADS / 32)
#define BW_WARP_DEFER_CAP (32 * BW_FOLD_UNROLL)
#define BW_NO_SLOT 0xFFFFFFFFu
// Staging of the rare global appends: common to every fold kernel.
struct DirtySink {
  u32 n_dirty;
  u32 n_new_keys;
  u32 cap;    // entries in buf
  u32* buf;   // shared-memory staging of dirty slot indices
};
struct BlockSinks : DirtySink {
  u32 dirty[BW_SINK_CAP];
  // per-warp queues of deferred events (arrival index within the batch)
  u32 n_defer[BW_FOLD_WARPS];
  u32 dq_g[BW_FOLD_WARPS][BW_WARP_DEFER_CAP];
  u32 dq_slot[BW_FOLD_WARPS][BW_WARP_DEFER_CAP];  // slot of the key when already known, else BW_NO_SLOT
};
__device__ __forceinline__ void bw_sinks_init(BlockSinks* sk) {
  if (threadIdx.x == 0) {
    sk->n_dirty = 0;
    sk->n_new_keys = 0;
    sk->cap = BW_SINK_CAP;
    sk->buf = sk->dirty;
  }
  if (threadIdx.x < BW_FOLD_WARPS) sk->n_defer[threadIdx.x] = 0;
}
// call by all threads of the block, after a __syncthreads()
__device__ __forceinline__ void bw_sinks_flush(DirtySink* sk, const Table& t) {
  __shared__ u32 base;
  u32 n = sk->n_dirty < sk->cap ? sk->n_dirty : sk->cap;
  if (threadIdx.x == 0) {
    base = n ? atomicAdd(&t.ctr->dirty_count, n) : 0u;
    if (sk->n_new_keys) atomicAdd(&t.ctr->live_keys, (unsigned long long)sk->n_new_keys);
  }
  __syncthreads();
  for (u32 i = threadIdx.x; i < n; i += blockDim.x) t.dirty[base + i] = sk->buf[i];
  __syncthreads();
  if (threadIdx.x == 0) {
    sk->n_dirty = 0;
    sk->n_new_keys = 0;
  }
  __syncthreads();
}

__device__ __forceinline__ u32 bw_ld_u32_coherent(const u32* p) {
  u32 v;
  asm volatile("ld.global.relaxed.gpu.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ i64 bw_ld_i64_coherent(const i64* p) {
  i64 v;
  asm volatile("ld.global.relaxed.gpu.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ u64 bw_home_slot(const Table& t, u64 key) {
  return (key == BW_EMPTY_KEY) ? t.cap : bw_slot_of_khash(bw_khash(key), t.cap);
}
// Linear probing wraps inside the segment of the home slot (Table::seg_mask): slot number `i`
// positions after `s` in probe order.
__device__ __forceinline__ u64 bw_probe_next(const Table& t, u64 s, u32 i) {
  return (s & ~(u64)t.seg_mask) | ((s + i) & (u64)t.seg_mask);
}

// Find (or create) the slot of `key`, starting at its home slot.  Four
// consecutive slots are fetched per round trip (independent sector loads), so a
// linear-probe chain costs ceil(len / 4) L2 latencies.  Returns ~0 on a full table.
#define BW_PROBE_WIDTH 4
__device__ __forceinline__ u64 bw_find_slot(const Table& t, DirtySink* sk, u64 key, i64& max_ts, i64& wt0) {
  u64 s = bw_home_slot(t, key);
  if (key == BW_EMPTY_KEY) {  // alias slot: always "found"
    u64 k, a;
    bw_ld_slot(t.hot + s, k, max_ts, wt0, a);
    return s;
  }
  for (u64 probe = 0; probe <= (u64)t.seg_mask;) {
    // four independent sector loads, then pick the first slot that holds the key or is free
    // (constant indices only: the probe state stays in registers)
    u64 k[BW_PROBE_WIDTH], a[BW_PROBE_WIDTH];
    i64 m[BW_PROBE_WIDTH], w[BW_PROBE_WIDTH];
#pragma unroll
    for (int j = 0; j < BW_PROBE_WIDTH; ++j) bw_ld_slot(t.hot + bw_probe_next(t, s, j), k[j], m[j], w[j], a[j]);
    int jm = BW_PROBE_WIDTH;
    u64 kk = 0;
    i64 mm = 0, ww = 0;
#pragma unroll
    for (int j = BW_PROBE_WIDTH - 1; j >= 0; --j) {
      if (k[j] == key || k[j] == BW_EMPTY_KEY) {
        jm = j;
        kk = k[j];
        mm = m[j];
        ww = w[j];
      }
    }
    if (jm == BW_PROBE_WIDTH) {
      s = bw_probe_next(t, s, BW_PROBE_WIDTH);
      probe += BW_PROBE_WIDTH;
      continue;
    }
    const u64 sj = bw_probe_next(t, s, (u32)jm);
    if (kk == key) {
      max_ts = mm;
      wt0 = ww;
      return sj;
    }
    HotSlot* hs = t.hot + sj;
    const u64 old = bw_key_claim(t, sj, key);
    if (old == BW_EMPTY_KEY) {
      // a free slot is always in the reset state; nobody else touches it before the key is set
      atomicAdd(&sk->n_new_keys, 1u);
      max_ts = mm;
      wt0 = ww;
      return sj;
    }
    if (old == key) {
      u64 k2, a2;
      bw_ld_slot(hs, k2, max_ts, wt0, a2);
      return sj;
    }
    // another key took it: resume right after it
    s = bw_probe_next(t, sj, 1);
    probe += (u64)jm + 1;
  }
  return ~0ULL;
}

__device__ __noinline__ void bw_mark_dirty(const Table& t, DirtySink* sk, u64 s) {
  unsigned long long old = atomicOr((unsigned long long*)&t.hot[s].wt0, (unsigned long long)BW_TAG_DIRTY);
  if (!(old & (unsigned long long)BW_TAG_DIRTY)) {
    u32 i = atomicAdd(&sk->n_dirty, 1u);
    if (i < sk->cap) {
      sk->buf[i] = (u32)s;
    } else {  // staging full: append directly
      u32 g = atomicAdd(&t.ctr->dirty_count, 1u);
      t.dirty[g] = (u32)s;
    }
  }
}

// Find or create the overflow pane node (key slot s, pane q).  Returns node index or 0 on failure.
__device__ __noinline__ u32 bw_spill_node(const Table& t, const FoldParams& p, u64 s, i64 q, u32 batch_no,
                                         bool& created) {
  AuxSlot* ax = t.aux + s;
  created = false;
  u32 n = bw_ld_u32_coherent(&ax->spill_head);
  while (n) {
    if (bw_ld_i64_coherent(&t.nodes[n].wid) == q) return n;
    n = bw_ld_u32_coherent(&t.nodes[n].next);
  }
  u32 result = 0;
  bool done = false;
  while (!done) {
    if (atomicCAS(&ax->lock, 0u, 1u) == 0u) {
      __threadfence();
      u32 head = bw_ld_u32_coherent(&ax->spill_head);
      n = head;
      while (n) {
        if (bw_ld_i64_coherent(&t.nodes[n].wid) == q) break;
        n = bw_ld_u32_coherent(&t.nodes[n].next);
      }
      if (!n) {
        int top = atomicSub(&t.ctr->free_top, 1);
        if (top > 0) {
          n = t.free_stack[top - 1];
        } else {
          atomicAdd(&t.ctr->free_top, 1);
          n = atomicAdd(&t.ctr->pool_next, 1u);
          if (n >= t.pool_cap) {
            n = 0;
            bw_raise(t.ctr, 3u /*BW_ERR_CAPACITY*/);
          }
        }
        if (n) {
          PaneNode nd;
          nd.wid = q;
          nd.acc = p.acc_identity;
          nd.open_seq = ~0ULL;
          nd.next = head;
          nd.born = batch_no;
          t.nodes[n] = nd;
          t.node_acc2[n] = 0;
          __threadfence();
          atomicExch(&ax->spill_head, n);
          if (!head) atomicOr((unsigned long long*)&t.hot[s].wt0, (unsigned long long)BW_TAG_HAS_LIST);
          created = true;
        }
      }
      result = n;
      __threadfence();
      atomicExch(&ax->lock, 0u);
      done = true;
    }
  }
  return result;
}

// Watermark tracking + "this key may have something to close / re-rank" marking.
// `q`, `rem` = pane and remainder of the event's own timestamp.  K4 leaves in
// the tag's delta field d = q0 - T where T is the pane-unit threshold of the
// key's earliest closable window; the event proves it closable iff
// q - close_back - (rem < wait_rem) >= q0 - d.  255 == "always re-examine".
template <class C>
__device__ __forceinline__ void bw_after_fold(const Table& t, const FoldParams& p, DirtySink* sk, u64 s, i64 ts,
                                              i64 mts, i64 tag0, bool created, i64 q, i64 rem) {
  HotSlot* hs = t.hot + s;
  if (C::wm(p)) {
    if (ts > mts) bw_red_max_s64(&hs->max_ts, ts);
    if (!(tag0 & BW_TAG_DIRTY)) {
      // (a moving system clock, FoldParams::now_us: the key's watermark also grew while it was idle, so what this
      // event's own timestamp proves closable is not the whole story: K4 looks at every key the activation touched)
      bool mark = created || p.now_us != 0;
      if (!mark) {
        const u32 delta = bw_widtag_delta(tag0);
        const i64 qc = q - p.close_back - ((rem < p.wait_rem) ? 1 : 0);
        mark = (delta == BW_TAG_DELTA_MAX) || (qc >= bw_widtag_q(tag0) - (i64)delta);
      }
      if (mark) bw_mark_dirty(t, sk, s);
    }
  } else if (created && !(tag0 & BW_TAG_DIRTY)) {
    bw_mark_dirty(t, sk, s);  // keep the newest panes in the direct slots for the next batch
  }
}

// merge a combined delta into a table accumulator
__device__ __forceinline__ void bw_merge(int op, u64* acc, u64 d) {
  if (op == BW_OP_ADD_ONE) bw_red_add_u64(acc, d);
  else bw_apply(op, acc, d);
}

// General path: any event (new key, displaced key, second / further pane).
// `seq` = (batch_no << 32) | arrival index.  PARTIAL: the "event" is a pre-combined partial
// (bw_stream.cuh: a delta of `weight` values whose newest timestamp is `ts`): the operand is
// merged instead of applied and the value count grows by `weight`.
template <class C, bool PARTIAL = false>
__device__ __noinline__ void bw_fold_event(const Table& t, const FoldParams& p, DirtySink* sk, u64 key, i64 ts,
                                           u64 operand, u64 seq, u32 batch_no, u32 known_slot, u64 weight = 1ULL) {
  i64 rem;
  const i64 q = bw_pane_of_r(ts, p, rem);
  if (q <= -BW_WID_LIMIT || q >= BW_WID_LIMIT) {
    bw_raise(t.ctr, 6u /*BW_ERR_RANGE*/);
    return;
  }
  i64 mts, tag0;
  u64 s;
  if (known_slot != BW_NO_SLOT) {
    u64 kk, aa;
    s = known_slot;
    bw_ld_slot(t.hot + s, kk, mts, tag0, aa);
  } else {
    s = bw_find_slot(t, sk, key, mts, tag0);
    if (s == ~0ULL) {
      bw_raise(t.ctr, 3u);
      return;
    }
  }
  HotSlot* hs = t.hot + s;
  const u32 born = batch_no & 63u;
  if (tag0 == BW_EMPTY_WIDTAG) {
    // delta = q - T, T = a * ceil((q - b + 1) / a): threshold of the first window covering this pane
    const i64 a = p.panes_per_offset, b = p.panes_per_window;
    const i64 d0 = (a == 1) ? (b - 1) : (q - a * bw_floordiv(q - b + a, a));
    i64 mine = bw_pack_widtag(q, d0 > (i64)BW_TAG_DELTA_MAX ? BW_TAG_DELTA_MAX : (u32)d0, born);
    i64 old = (i64)atomicCAS((unsigned long long*)&hs->wt0, (unsigned long long)BW_EMPTY_WIDTAG, (unsigned long long)mine);
    tag0 = (old == BW_EMPTY_WIDTAG) ? mine : old;
  }
  const int op = C::op(p);
  bool created = false;
  if (bw_widtag_q(tag0) == q) {
    if (PARTIAL) bw_merge(op, &hs->acc0, operand);
    else bw_apply(op, &hs->acc0, operand);
    if (C::cnt(p)) bw_red_add_u64(&t.aux[s].cnt0, weight);
    if (((u32)tag0 & 0x7Fu) == born) bw_red_min_u64(&t.aux[s].seq0, seq);
  } else if (bw_widtag_q1(tag0) == q) {
    if (PARTIAL) bw_merge(op, &t.p1[s].acc1, operand);
    else bw_apply(op, &t.p1[s].acc1, operand);
    if (!(tag0 & BW_TAG_P1_PREV)) bw_red_min_u64(&t.p1[s].seq1, seq);  // presence + first-open order
    if (!(tag0 & BW_TAG_HAS_P1)) atomicOr((unsigned long long*)&hs->wt0, (unsigned long long)BW_TAG_HAS_P1);
    if (C::cnt(p)) bw_red_add_u64(&t.aux[s].cnt1, weight);
  } else {
    u32 n = bw_spill_node(t, p, s, q, batch_no, created);
    if (!n) return;
    if (PARTIAL) bw_merge(op, &t.nodes[n].acc, operand);
    else bw_apply(op, &t.nodes[n].acc, operand);
    if (C::cnt(p)) bw_red_add_u64(&t.node_acc2[n], weight);
    if (t.nodes[n].born == batch_no) bw_red_min_u64(&t.nodes[n].open_seq, seq);
  }
  bw_after_fold<C>(t, p, sk, s, ts, mts, tag0, created, q, rem);
}

__device__ __forceinline__ void bw_operand(const FoldParams& p, u64 raw, u64& operand);

// Read-only lookup of a key that is not in its home slot (about a third of the keys at load
// 0.5): the same 4-wide probe as bw_find_slot without the claim logic.  Returns BW_NO_SLOT when
// the probe reaches a free slot (new key) or the window is exhausted: those go to bw_fold_event.
__device__ __forceinline__ u32 bw_lookup_slot(const Table& t, u64 key, i64& max_ts, i64& wt0) {
  u64 s = bw_home_slot(t, key);
  if (key == BW_EMPTY_KEY) return BW_NO_SLOT;
#pragma unroll 1
  for (int round = 0; round < 4; ++round) {
    u64 k[BW_PROBE_WIDTH], a[BW_PROBE_WIDTH];
    i64 m[BW_PROBE_WIDTH], w[BW_PROBE_WIDTH];
#pragma unroll
    for (int j = 0; j < BW_PROBE_WIDTH; ++j) bw_ld_slot(t.hot + bw_probe_next(t, s, j), k[j], m[j], w[j], a[j]);
    int jm = BW_PROBE_WIDTH;
    u64 kk = 0;
    i64 mm = 0, ww = 0;
#pragma unroll
    for (int j = BW_PROBE_WIDTH - 1; j >= 0; --j) {
      if (k[j] == key || k[j] == BW_EMPTY_KEY) {
        jm = j;
        kk = k[j];
        mm = m[j];
        ww = w[j];
      }
    }
    if (jm < BW_PROBE_WIDTH) {
      if (kk != key) return BW_NO_SLOT;
      max_ts = mm;
      wt0 = ww;
      return (u32)bw_probe_next(t, s, (u32)jm);
    }
    s = bw_probe_next(t, s, BW_PROBE_WIDTH);
  }
  return BW_NO_SLOT;
}

// The common case, given the slot of a known key and the sector read from it: the event falls in
// the key's pane 0 or pane 1.  Applies it to the table and returns true; returns false for every other case.
template <class C>
__device__ __forceinline__ bool bw_try_fast(const Table& t, const FoldParams& p, DirtySink* sk, u32 slot, i64 tag0, i64 mts,
                                            i64 ts, u64 raw, u64 seq, u32 born, PaneCache& pc) {
  i64 rem;
  const i64 q = bw_pane_cached(ts, p, rem, pc);
  const bool usable = tag0 != BW_EMPTY_WIDTAG && (q > -BW_WID_LIMIT) && (q < BW_WID_LIMIT);
  const bool hit0 = usable && bw_widtag_q(tag0) == q;
  const bool hit1 = usable && !hit0 && bw_widtag_q1(tag0) == q;
  if (!(hit0 || hit1)) return false;
  u64 operand;
  bw_operand(p, raw, operand);
  if (hit0) {
    bw_apply(C::op(p), &t.hot[slot].acc0, operand);
    if (C::cnt(p)) bw_red_add_u64(&t.aux[slot].cnt0, 1ULL);
    if (((u32)tag0 & 0x7Fu) == born) bw_red_min_u64(&t.aux[slot].seq0, seq);
  } else {
    P1Slot* ps = t.p1 + slot;
    bw_apply(C::op(p), &ps->acc1, operand);
    if (!(tag0 & BW_TAG_P1_PREV)) bw_red_min_u64(&ps->seq1, seq);
    if (!(tag0 & BW_TAG_HAS_P1)) atomicOr((unsigned long long*)&t.hot[slot].wt0, (unsigned long long)BW_TAG_HAS_P1);
    if (C::cnt(p)) bw_red_add_u64(&t.aux[slot].cnt1, 1ULL);
  }
  bw_after_fold<C>(t, p, sk, slot, ts, mts, tag0, false, q, rem);
  return true;
}

// raw value bits -> accumulator operand
__device__ __forceinline__ void bw_operand(const FoldParams& p, u64 raw, u64& operand) {
  if (p.val_dtype >= 2) {
    double d = (p.val_dtype == 2) ? (double)__uint_as_float((u32)raw) : __longlong_as_double((i64)raw);
    u64 b = (u64)__double_as_longlong(d);
    operand = (p.op == BW_OP_ADD_F64) ? b : bw_f64_to_ordered(b);
  } else {
    operand = raw;
    if (p.op == BW_OP_ADD_F64) {  // MEAN over integers accumulates in f64
      double d = (p.val_dtype == 1) ? (double)(i64)raw : (double)raw;
      operand = (u64)__double_as_longlong(d);
    }
  }
}

// value bits -> accumulator operand, and the event time
__device__ __forceinline__ void bw_load_event(const BatchView& bv, int seg, u64 i, const FoldParams& p, u64& key,
                                              i64& ts, u64& operand, u64& raw) {
  key = bw_ld_stream_u64(bv.keys[seg] + i);
  raw = 0;
  if (bv.vals[seg]) {
    if (p.val_dtype == 2 /*F32*/) {
      raw = bw_ld_stream_u32((const u32*)bv.vals[seg] + i);
    } else {
      raw = bw_ld_stream_u64((const u64*)bv.vals[seg] + i);
    }
  }
  if (p.ts_from_value) {
    ts = p.align_us + ((p.ts_from_value == 1) ? (i64)raw : 0);  // 2 == BW_TS_NONE: everything in window 0
  } else {
    ts = (i64)bw_ld_stream_u64((const u64*)bv.ts[seg] + i) - p.now_us;
  }
  // operand in accumulator representation
  if (p.val_dtype >= 2) {
    double d = (p.val_dtype == 2) ? (double)__uint_as_float((u32)raw) : __longlong_as_double((i64)raw);
    u64 b = (u64)__double_as_longlong(d);
    operand = (p.op == BW_OP_ADD_F64) ? b : bw_f64_to_ordered(b);
  } else {
    operand = raw;
    if (p.op == BW_OP_ADD_F64) {  // MEAN over integers accumulates in f64
      double d = (p.val_dtype == 1) ? (double)(i64)raw : (double)raw;
      operand = (u64)__double_as_longlong(d);
    }
  }
}

// Map a global arrival index to (segment, offset).
__device__ __noinline__ bool bw_locate(const BatchView& bv, const u64* seg_start, u64 g, int& seg, u64& off) {
  seg = 0;
#pragma unroll
  for (int j = 1; j < BW_MAX_WORLD; ++j)
    if (j < bv.nseg && g >= seg_start[j]) seg = j;
  off = g - seg_start[seg];
  return true;
}

// Event time of arrival index g (value-derived, or re-read from the ts column: an L1/L2 hit).
__device__ __forceinline__ i64 bw_event_ts(const BatchView& bv, const u64* seg_start, const FoldParams& p, u64 g,
                                           u64 raw) {
  if (p.ts_from_value) return p.align_us + ((p.ts_from_value == 1) ? (i64)raw : 0);
  int seg = 0;
  u64 off = g;
  if (bv.nseg > 1) bw_locate(bv, seg_start, g, seg, off);
  return (i64)bw_ld_stream_u64((const u64*)bv.ts[seg] + off) - p.now_us;
}

// The fold kernel.  Launched only for batches the prepass proved free of late
// items (or when the clock never advances on data, wait == forever).
template <class C>
__global__ void __launch_bounds__(BW_FOLD_THREADS, BW_FOLD_MINB)
k_fold(BatchView bv, Table t, FoldParams p, u32 batch_no, u32 sub_i, u32 sub_n) {
  __shared__ u64 seg_start[BW_MAX_WORLD + 1];
  __shared__ BlockSinks sinks;
  bw_sinks_init(&sinks);
  if (threadIdx.x == 0) {
    u64 acc = 0;
    for (int j = 0; j < bv.nseg; ++j) {
      seg_start[j] = acc;
      acc += bw_seg_count(bv, j);
    }
    seg_start[bv.nseg] = acc;
  }
  __syncthreads();
  // sub-range sub_i of sub_n of the activation, by arrival index (the caller closes between
  // sub-ranges so that a key moving through several windows keeps hitting the two direct panes)
  const u64 all = seg_start[bv.nseg];
  const u64 range_lo = (sub_n > 1) ? (all * sub_i) / sub_n : 0;
  const u64 total = (sub_n > 1) ? (all * (sub_i + 1ULL)) / sub_n : all;
  const u64 tile = (u64)BW_FOLD_THREADS * BW_FOLD_UNROLL;
  const u32 born = batch_no & 63u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  u32 iter = 0;
  PaneCache pcache;
  pcache.lo = INT64_MAX;
  pcache.q = 0;
  for (u64 base = range_lo + (u64)blockIdx.x * tile; base < total; base += (u64)gridDim.x * tile) {
    // a warp owns BW_FOLD_UNROLL runs of 32 consecutive events
    const u64 wbase = base + (u64)warp * (32 * BW_FOLD_UNROLL);
    // after an exchange the activation is up to 8 segments: resolve the segment once per warp-run
    // when the whole run lies inside one (all but <= 7 runs of a launch do)
    int wseg = 0;
    bool wuni = true;
    if (bv.nseg > 1) {
      const u64 wlast = (wbase + 32 * BW_FOLD_UNROLL - 1 < total) ? wbase + 32 * BW_FOLD_UNROLL - 1 : total - 1;
#pragma unroll
      for (int j = 1; j < BW_MAX_WORLD; ++j)
        if (j < bv.nseg && wbase >= seg_start[j]) wseg = j;
      wuni = (wseg + 1 >= bv.nseg) || (wlast < seg_start[wseg + 1]);
    }
    u64 key[BW_FOLD_UNROLL], raw[BW_FOLD_UNROLL];
    // phase A: stream the events in, then issue every home-slot read before using any
#pragma unroll
    for (int u = 0; u < BW_FOLD_UNROLL; ++u) {
      const u64 g = wbase + (u64)u * 32 + lane;
      key[u] = 0;
      raw[u] = 0;
      if (g < total) {
        int seg = wseg;
        u64 off = g - seg_start[wseg];
        if (!wuni) bw_locate(bv, seg_start, g, seg, off);
        key[u] = bw_ld_stream_u64(bv.keys[seg] + off);
        if (p.ts_from_value == 1 || bv.vals[seg]) {
          raw[u] = (p.val_dtype == 2) ? (u64)bw_ld_stream_u32((const u32*)bv.vals[seg] + off)
                                      : bw_ld_stream_u64((const u64*)bv.vals[seg] + off);
        }
      }
    }
    u64 k0[BW_FOLD_UNROLL], a0[BW_FOLD_UNROLL];
    i64 mts[BW_FOLD_UNROLL], tag0[BW_FOLD_UNROLL];
    u32 slot[BW_FOLD_UNROLL];
#pragma unroll
    for (int u = 0; u < BW_FOLD_UNROLL; ++u) {
      slot[u] = (u32)bw_home_slot(t, key[u]);
      bw_ld_slot(t.hot + slot[u], k0[u], mts[u], tag0[u], a0[u]);
    }
    // phase B: events in the key's pane 0 or pane 1 finish here from the one
    // sector already read; everything else goes to the warp's queue.
#pragma unroll
    for (int u = 0; u < BW_FOLD_UNROLL; ++u) {
      const u64 g = wbase + (u64)u * 32 + lane;
      if (g >= total) continue;
      const i64 ts = bw_event_ts(bv, seg_start, p, g, raw[u]);
      const bool known = (k0[u] == key[u]);
      if (!(known && bw_try_fast<C>(t, p, &sinks, slot[u], tag0[u], mts[u], ts, raw[u],
                                           ((u64)batch_no << 32) | g, born, pcache))) {
        u32 i = atomicAdd(&sinks.n_defer[warp], 1u);
        sinks.dq_g[warp][i] = (u32)g;
        sinks.dq_slot[warp][i] = known ? slot[u] : BW_NO_SLOT;
      }
    }
    __syncwarp();
    // phase C: the warp drains its own queue with dense lanes (no block barrier).  Most of the
    // queue is known keys that simply do not sit in their home slot: a read-only probe plus the
    // same fast apply; only new keys and third panes need the general path.
    const u32 nd = sinks.n_defer[warp];
    for (u32 i = lane; i < nd; i += 32) {
      const u64 g = sinks.dq_g[warp][i];
      int seg = 0;
      u64 off = g;
      if (bv.nseg > 1) bw_locate(bv, seg_start, g, seg, off);
      u64 kk, op, rw;
      i64 ts;
      bw_load_event(bv, seg, off, p, kk, ts, op, rw);
      const u64 seq = ((u64)batch_no << 32) | g;
      u32 ks = sinks.dq_slot[warp][i];
      if (ks == BW_NO_SLOT) {
        i64 m2, w2;
        ks = bw_lookup_slot(t, kk, m2, w2);
        if (ks != BW_NO_SLOT && bw_try_fast<C>(t, p, &sinks, ks, w2, m2, ts, rw, seq, born, pcache)) continue;
      }
      bw_fold_event<C>(t, p, &sinks, kk, ts, op, seq, batch_no, ks);
    }
    __syncwarp();
    if (lane == 0) sinks.n_defer[warp] = 0;
    __syncwarp();
    // the staged dirty list is flushed block-wide now and then (it overflows safely
    // to direct appends, so this is only about keeping the global cursor cold)
    if ((++iter & 7u) == 0u) {
      __syncthreads();
      if (sinks.n_dirty > BW_SINK_CAP / 4) bw_sinks_flush(&sinks, t);  // uniform: read after the barrier
    }
  }
  __syncthreads();
  bw_sinks_flush(&sinks, t);
}
