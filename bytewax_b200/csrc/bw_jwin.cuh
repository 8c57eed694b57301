// bw_jwin.cuh -- K8: `join_window` with insert modes first / last over tumbling and sliding windows.
//
// The reference runs `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) over
// `_SlidingWindowerLogic` (:603-668) with one `_JoinWindowLogic` (:1849-1902) per window: per key, in arrival order,
// the EventClock's late test; the queue; `_flush_queue` (:1095-1108), which in ordered mode plays the entries with
// ts <= watermark in timestamp order (stable) and keeps the rest queued; the join step per window; the close in
// first-opened order.  All of it depends on order, so the device does what K6 / K7 do: values travel as u64 handles,
// the activation is grouped by key (CUB stable sort, `keyed_group`), and ONE thread per key restates the steps.
//
// Unordered mode: one kernel per activation (k_jwin_apply) walks a key's items twice: the late test, then the play of
// the on-time items in arrival order, then the close.
// Ordered mode: k_jwin_apply does the late test and appends the on-time items to the key's queue; the queue of every
// key lives in one pool.  Then the due entries are put in play order by two stable CUB radix sorts over the pool --
// (ts of a due entry, or ~0 for one that stays queued) and then the key's slot -- so no thread sorts; k_jwin_flush,
// one thread per slot, plays its key's due entries, carries the rest over to the next pool in their order, and closes.
// Notify and EOF mark the keys they wake (k_jwin_mark) and run the same flush.
//
// Handles are released (bw_jwin_rows.released) in the call in which no window and no queue entry of their key holds
// them any more: a late item's at once, a "first" value that found its side set, a value replaced by "last" or cleared
// by "complete", and a window's values when it closes -- each only once no other window of the key holds it.
//
// Per key:
//   keys[slot]            the key (bw_keyed_find table; slot `cap` is the BW_EMPTY_KEY alias slot)
//   st[slot]              the EventClock pair, the watermark and call of the current flush, open windows n, queued
//                         entries nq and the ts of the first one, the key's range in the sorted pool
//   win[slot * M ...]     open windows in first-opened order (the reference's dict order): id, set mask, handles
// The pool (ordered mode): slot, ts, handle, side per entry; a key's entries in arrival order.
#pragma once
#include "../../include/bwgpu.h"
#include "bw_common.cuh"
#include "bw_keyed.cuh"

#define BW_JW_MAXM 64
#define BW_JW_MAXSIDES 4
#define BW_JW_DROP 0xFF  // pool entry of a late item: not queued
// reasons behind a BW_ERR_CAPACITY, or-ed into JwTable::why
enum { BW_JW_FULL_TABLE = 1, BW_JW_FULL_WINDOWS = 2, BW_JW_FULL_EMIT = 4, BW_JW_FULL_LATE = 8, BW_JW_FULL_QUEUE = 16, BW_JW_BAD_SIDE = 32 };

struct JwState {
  i64 wm_base;  // _EventClockState.watermark_base
  i64 sys_max;  // _EventClockState.system_time_of_max_event
  i64 wm;       // watermark of the flush of call `act`
  i64 q0ts;     // ts of queue[0] (notify_at, windowing.py:1163-1168)
  u64 act;      // call ordinal of the last flush that woke the key
  u64 qord;     // call ordinal of [qb, qe): the key's range of the sorted pool
  u32 qb, qe;
  u32 n, nq;    // open windows, queued entries
  u32 init, pad;
};
struct __align__(16) JwWin {
  i64 id;
  u64 mask;
  u64 h[BW_JW_MAXSIDES];
  __device__ void open(i64 i) {
    id = i;
    mask = 0;
  }
};
struct JwTable {
  u64* keys;
  JwState* st;
  JwWin* win;
  u64 cap;
  int M, sides;
  u32* err;  // BW_ERR_CAPACITY once anything overflowed (BW_ERR_SPEC: a side column value >= sides)
  u32* why;  // BW_JW_FULL_* / BW_JW_BAD_SIDE bits
};
struct JwPool {  // entries in arrival order per key
  u32* slot;
  i64* ts;
  u64* h;
  unsigned char* side;
};
struct JwEmit {
  // down: joined tuples
  u64 *key, *wid, *h0, *h1, *h2, *h3, *mask, *epoch, *ord, *seq;
  u64 max_rows;
  unsigned long long* n_rows;
  // meta: closed windows
  u64 *m_key, *m_wid, *m_epoch, *m_ord, *m_seq;
  unsigned long long* n_meta;
  // late items, one row per window id
  u64 *l_key, *l_wid, *l_epoch, *l_act, *l_row, *l_ord, *l_seq;
  u64 max_late;
  unsigned long long* n_late;
  // released handles
  u64* rel;
  u64 max_rel;
  unsigned long long* n_rel;
  // ordered mode: entries carried over to the next pool
  JwPool next;
  u64 max_queue;
  unsigned long long* n_next;
};
struct JwParams {
  int insert_last, emit_mode, ordered;
  i64 length, offset, align, wait, now;
  u64 epoch, ord;
  u32 batch_no;
};

// (T, E: JwTable / JwEmit here, and the tables and emit buffers of the kernels that share these steps, bw_collect.cuh)
template <class T>
__device__ __forceinline__ void bw_jw_fail(const T& t, u32 bit) {
  atomicOr(t.why, bit);
  atomicCAS(t.err, 0u, (u32)BW_ERR_CAPACITY);
}

// a device column named a side >= sides: the item is dropped unplayed and the call fails
__device__ __forceinline__ void bw_jw_bad_side(const JwTable& t) {
  atomicOr(t.why, (u32)BW_JW_BAD_SIDE);
  atomicCAS(t.err, 0u, (u32)BW_ERR_SPEC);
}

__device__ __forceinline__ i64 bw_jw_floordiv(i64 a, i64 b) {  // b > 0
  i64 q = a / b;
  return (a % b != 0 && a < 0) ? q - 1 : q;
}
// intersects(ts), windowing.py:611-618: ids lo..hi (hi < lo: none)
__device__ __forceinline__ void bw_jw_ids(const JwParams& p, i64 ts, i64& lo, i64& hi) {
  const i64 since = ts - p.align;
  lo = bw_jw_floordiv(since - p.length, p.offset) + 1;
  hi = bw_jw_floordiv(since, p.offset);
}
__device__ __forceinline__ i64 bw_jw_close(const JwParams& p, i64 id) { return p.align + p.offset * id + p.length; }

// the window `id` among a key's n open windows W (first-opened order), opened at the end when absent (`open_for`: a
// window is opened on its first value); M when the key already holds M windows
template <class W>
__device__ __forceinline__ u32 bw_jw_find_or_open(W* Ws, u32& n, u32 M, i64 id) {
  u32 i = 0;
  while (i < n && Ws[i].id != id) ++i;
  if (i == n) {
    if (n >= M) return M;
    Ws[n].open(id);
    ++n;
  }
  return i;
}

// `_handle_closed` (windowing.py:1087-1093): every window with close <= wm leaves W in first-opened order; `on_close`
// sees it after it has left (so W[0, n) are the windows still open)
template <class W, class F>
__device__ __forceinline__ void bw_jw_close_each(const JwParams& p, W* Ws, u32& n, i64 wm, F&& on_close) {
  u32 i = 0;
  while (i < n) {
    if (bw_jw_close(p, Ws[i].id) > wm) {
      ++i;
      continue;
    }
    const W w = Ws[i];
    for (u32 j = i + 1; j < n; ++j) Ws[j - 1] = Ws[j];
    --n;
    on_close(w);
  }
}

// builder(None) of a key with no logic: _EventClockLogic.__post_init__ (windowing.py:245-248), empty windower and queue
__device__ __forceinline__ void bw_jw_begin(JwState& st, const JwParams& p) {
  if (st.init) return;
  st.init = 1;
  st.wm_base = BW_UTC_MIN_US;
  st.sys_max = p.now;
  st.n = st.nq = 0;
  st.qord = ~0ULL;
}

// _EventClockLogic.on_item (windowing.py:263-287; ts - wait below UTC_MIN raises OverflowError: ignored): the watermark
// after the item goes to wm; true when the item is late
__device__ __forceinline__ bool bw_jw_on_item(JwState& st, const JwParams& p, i64 ts, i64& wm) {
  wm = st.wm_base + (p.now - st.sys_max);
  if (p.wait != BW_WAIT_FOREVER && ts - BW_UTC_MIN_US >= p.wait) {
    const i64 cand = ts - p.wait;
    if (cand > wm) {
      st.wm_base = cand;
      st.sys_max = p.now;
      wm = cand;
    }
  }
  return ts < wm;
}

// a late item: one row per id of intersects(ts), ascending (windowing.py:636-637, :1125-1127), naming input row o
template <class T, class E>
__device__ void bw_jw_late_rows(const T& t, const E& e, const JwParams& p, u64 key, i64 ts, u32 o, u64& lseq) {
  i64 lo, hi;
  bw_jw_ids(p, ts, lo, hi);
  const u64 cnt = hi >= lo ? (u64)(hi - lo + 1) : 0;
  const u64 i0 = cnt > e.max_late ? e.max_late : atomicAdd(e.n_late, (unsigned long long)cnt);
  if (i0 + cnt > e.max_late) {
    bw_jw_fail(t, BW_JW_FULL_LATE);
    return;
  }
  for (u64 c = 0; c < cnt; ++c) {
    e.l_key[i0 + c] = key;
    e.l_wid[i0 + c] = (u64)(lo + (i64)c);
    e.l_epoch[i0 + c] = p.epoch;
    e.l_act[i0 + c] = p.batch_no;
    e.l_row[i0 + c] = o;
    e.l_ord[i0 + c] = p.ord;
    e.l_seq[i0 + c] = lseq++;
  }
}

template <class T, class E>
__device__ __forceinline__ void bw_jw_release(const T& t, const E& e, u64 h) {
  const u64 i = atomicAdd(e.n_rel, 1ULL);
  if (i < e.max_rel) e.rel[i] = h;  // (the host sizes the buffer for every handle the call can release: never reached)
  else bw_jw_fail(t, BW_JW_FULL_EMIT);
}
// does any of the key's n windows hold h
__device__ __forceinline__ bool bw_jw_held(const JwWin* W, u32 n, int sides, u64 h) {
  for (u32 i = 0; i < n; ++i)
    for (int s = 0; s < sides; ++s)
      if ((W[i].mask >> s & 1) && W[i].h[s] == h) return true;
  return false;
}

__device__ void bw_jw_emit(const JwTable& t, const JwEmit& e, const JwParams& p, u64 key, const JwWin& w, u64& seq) {
  const u64 row = atomicAdd(e.n_rows, 1ULL);
  if (row >= e.max_rows) {
    bw_jw_fail(t, BW_JW_FULL_EMIT);
    return;
  }
  e.key[row] = key;
  e.wid[row] = (u64)w.id;
  e.h0[row] = w.h[0];
  e.h1[row] = w.h[1];
  e.h2[row] = w.h[2];
  e.h3[row] = w.h[3];
  e.mask[row] = w.mask;
  e.epoch[row] = p.epoch;
  e.ord[row] = p.ord;
  e.seq[row] = seq++;
}

// one due entry: `_handle_inserts` (windowing.py:1064-1077) + `_JoinWindowLogic.on_value` (:1866-1876); false when
// the key needs more than M windows
__device__ bool bw_jw_play(const JwTable& t, const JwEmit& e, const JwParams& p, u64 key, JwWin* W, u32& n, i64 ts, u64 h, int side,
                           u64& seq) {
  const int sides = t.sides;
  const u64 full = (1ULL << sides) - 1, bit = 1ULL << side;
  i64 lo, hi;
  bw_jw_ids(p, ts, lo, hi);
  for (i64 id = lo; id <= hi; ++id) {
    const u32 i = bw_jw_find_or_open(W, n, (u32)t.M, id);
    if (i == (u32)t.M) return false;
    JwWin& w = W[i];
    if (!(w.mask & bit)) {
      w.h[side] = h;
      w.mask |= bit;
    } else if (p.insert_last) {
      const u64 old = w.h[side];
      w.h[side] = h;
      if (old != h && !bw_jw_held(W, n, sides, old)) bw_jw_release(t, e, old);
    }
    if (p.emit_mode == BW_JOIN_EMIT_COMPLETE) {
      if (w.mask == full) {
        bw_jw_emit(t, e, p, key, w, seq);
        w.mask = 0;  // _JoinState.clear
        for (int s = 0; s < sides; ++s)
          if (w.h[s] != h && !bw_jw_held(W, n, sides, w.h[s])) bw_jw_release(t, e, w.h[s]);
      }
    } else if (p.emit_mode == BW_JOIN_EMIT_RUNNING) {
      bw_jw_emit(t, e, p, key, w, seq);
    }
  }
  if (!bw_jw_held(W, n, sides, h)) bw_jw_release(t, e, h);  // never stored, or no longer
  return true;
}

// `_handle_closed` (windowing.py:1087-1093): windows with close <= watermark in first-opened order; `final` row, then meta
__device__ void bw_jw_close_windows(const JwTable& t, const JwEmit& e, const JwParams& p, u64 key, JwWin* W, u32& n, i64 wm, u64& seq,
                                    u64& mseq) {
  bw_jw_close_each(p, W, n, wm, [&](const JwWin& w) {
    if (p.emit_mode == BW_JOIN_EMIT_FINAL) bw_jw_emit(t, e, p, key, w, seq);
    const u64 m = atomicAdd(e.n_meta, 1ULL);
    if (m >= e.max_rows) {
      bw_jw_fail(t, BW_JW_FULL_EMIT);
    } else {
      e.m_key[m] = key;
      e.m_wid[m] = (u64)w.id;
      e.m_epoch[m] = p.epoch;
      e.m_ord[m] = p.ord;
      e.m_seq[m] = mseq++;
    }
    for (int s = 0; s < t.sides; ++s)
      if ((w.mask >> s & 1) && !bw_jw_held(W, n, t.sides, w.h[s])) bw_jw_release(t, e, w.h[s]);
  });
}

// notify_at (windowing.py:1153-1180), identity `to_system_utc`
template <class W>
__device__ __forceinline__ i64 bw_jw_notify_at(const JwParams& p, const JwState& st, const W* Ws) {
  i64 at = INT64_MAX;
  for (u32 i = 0; i < st.n; ++i) {
    const i64 c = bw_jw_close(p, Ws[i].id);
    at = c < at ? c : at;
  }
  if (p.ordered && st.nq && st.q0ts < at) at = st.q0ts;
  return at;
}

// pass A, one thread per key segment: the late test per item (windowing.py:1115-1133, :263-287).  Unordered: then the
// play of the on-time items in arrival order and the close.  Ordered: the on-time items go to the pool at base + q.
__global__ void k_jwin_apply(JwTable t, JwEmit e, JwParams p, JwPool pool, u64 base, const u64* ksorted, const u32* isorted,
                             const u32* headpos, const u64* handles, const unsigned char* sides, const i64* ts_us, unsigned char* late,
                             u64 n) {
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.keys, t.cap, key, t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      // the call fails, but the pool sort and flush that follow still read every entry of this call: the key's go in as
      // late items' entries under a valid slot, so they are neither played nor carried over
      for (u64 q = h; q < n && ksorted[q] == key; ++q)
        if (p.ordered) {
          pool.slot[base + q] = (u32)t.cap;
          pool.side[base + q] = (unsigned char)BW_JW_DROP;
        }
      continue;
    }
    JwState st = t.st[s];
    bw_jw_begin(st, p);
    u64 end = h;
    while (end < n && ksorted[end] == key) ++end;
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0;
    bool full = false;
    for (u64 q = h; q < end; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      if (sides[o] >= t.sides) {  // (device columns are not checked on the host)
        bw_jw_bad_side(t);
        if (p.ordered) {
          pool.slot[base + q] = (u32)s;
          pool.side[base + q] = (unsigned char)BW_JW_DROP;
        } else {
          late[q] = 1;
        }
        continue;
      }
      const bool is_late = bw_jw_on_item(st, p, ts, wm);
      if (is_late) {  // the late rows; the handle is let go
        bw_jw_late_rows(t, e, p, key, ts, o, lseq);
        bw_jw_release(t, e, handles[o]);
      }
      if (p.ordered) {
        pool.slot[base + q] = (u32)s;
        pool.ts[base + q] = ts;
        pool.h[base + q] = handles[o];
        pool.side[base + q] = is_late ? (unsigned char)BW_JW_DROP : sides[o];
      } else {
        late[q] = is_late;
      }
    }
    st.wm = wm;
    st.act = p.ord;
    if (!p.ordered) {  // every queued entry is due, in arrival order
      JwWin* W = t.win + s * (u64)t.M;
      u64 seq = 0, mseq = 0;
      u32 nw = st.n;
      for (u64 q = h; q < end && !full; ++q) {
        if (late[q]) continue;
        const u32 o = isorted[q];
        full = !bw_jw_play(t, e, p, key, W, nw, ts_us[o], handles[o], sides[o], seq);
      }
      if (full) {
        bw_jw_fail(t, BW_JW_FULL_WINDOWS);
        continue;  // the call fails and the join refuses further work: no row of this key is emitted half-done
      }
      bw_jw_close_windows(t, e, p, key, W, nw, wm, seq, mseq);
      st.n = nw;
      if (nw == 0) st.init = 0;  // _is_empty (windowing.py:1110-1113): the engine discards the logic, clock included
    }
    t.st[s] = st;
  }
}

// K8 on world > 1, at the owner: the received segments (bv.h_counts rows from each source) into K8's columns in (source
// rank, source order), the arrival order a world-1 join sees when it is fed the rank-major concatenation.  The handle
// travels in the value column, the side in the region's side column; name[i] = source rank << 32 | the row's index in
// that source's columns (src_row, src_side: the region's row and side columns, `cap` rows per source).
__global__ void k_xjwin_gather(BatchView bv, const u32* src_row, const unsigned char* src_side, u64 cap, u64 n, u64* keys, u64* handles,
                               unsigned char* side, i64* ts, u64* name) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    int r = 0;
    u64 o = i;
    while (o >= bv.h_counts[r]) o -= bv.h_counts[r++];
    keys[i] = bv.keys[r][o];
    handles[i] = ((const u64*)bv.vals[r])[o];
    side[i] = src_side[(u64)r * cap + o];
    ts[i] = bv.ts[r][o];
    name[i] = (u64)r << 32 | src_row[(u64)r * cap + o];
  }
}

// After k_jwin_apply on world > 1: the late rows this call added, [*before, *n_late), hold positions in the gathered
// columns (below n); give them their rows' names instead.  Names grow with the position, so arrival order holds.  A
// late item reserves one row per window id, all or none (bw_jw_late_rows): when a reservation crossed max_late, the
// slots it left unwritten still hold an earlier call's names, so nothing is renamed -- the call has failed
// (BW_JW_FULL_LATE) and its late rows are never handed out.
__global__ void k_xjwin_name_late(const unsigned long long* before, const unsigned long long* n_late, u64 max_late, u64* l_row,
                                  const u64* name, u64 n) {
  if (*n_late > max_late) return;
  for (u64 i = *before + (u64)blockIdx.x * blockDim.x + threadIdx.x; i < *n_late; i += (u64)gridDim.x * blockDim.x) {
    const u64 p = l_row[i];
    if (p < n) l_row[i] = name[p];  // (always, when no reservation failed)
  }
}

// notify_at of the sliding windower's keys (the default of k_jwin_mark)
struct JwNotifyAt {
  template <class W>
  __device__ __forceinline__ i64 operator()(const JwParams& p, const JwState& st, const W* Ws) const {
    return bw_jw_notify_at(p, st, Ws);
  }
};

// notify (src/operators.rs:808-858): keys whose notify_at has come, at the watermark `on_notify` sees (:289-298);
// EOF (:862-894, windowing.py:1144-1151): every key, watermark UTC_MAX
// (W: the table's window records, JwWin here; N: the windower's notify_at, JwNotifyAt here, SjNotifyAt for sessions)
template <class W, class N = JwNotifyAt>
__global__ void k_jwin_mark(JwTable t, const W* win, JwParams p, int eof, N notify_at = N()) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    JwState& st = t.st[s];
    if (!st.init) continue;
    if (eof) {
      st.wm = BW_UTC_MAX_US;
    } else {
      if (notify_at(p, st, win + s * (u64)t.M) > p.now) continue;
      st.wm = st.wm_base + (p.now - st.sys_max);
    }
    st.act = p.ord;
  }
}

// sort key of pool entry i: its ts when it is due in this flush, ~0 when it stays queued (or is a late item's)
__global__ void k_jwin_sortkey(JwTable t, JwParams p, JwPool pool, u64* sk, u32* perm, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const JwState& st = t.st[pool.slot[i]];
    const bool due = pool.side[i] != BW_JW_DROP && st.act == p.ord && pool.ts[i] <= st.wm;
    sk[i] = due ? (u64)pool.ts[i] ^ (1ULL << 63) : ~0ULL;
    perm[i] = (u32)i;
  }
}
__global__ void k_jwin_slotkey(JwPool pool, const u32* perm, u64* sk, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) sk[i] = pool.slot[perm[i]];
}
// every key's range of the sorted pool
__global__ void k_jwin_ranges(JwTable t, JwParams p, JwPool pool, const u32* perm, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const u32 s = pool.slot[perm[i]];
    if (i == 0 || pool.slot[perm[i - 1]] != s) {
      u64 j = i + 1;
      while (j < n && pool.slot[perm[j]] == s) ++j;
      t.st[s].qb = (u32)i;
      t.st[s].qe = (u32)j;
      t.st[s].qord = p.ord;
    }
  }
}

// the `keep` entries of slot s's range [qb, qe) of the sorted pool that are not due stay queued, in their order
// (windowing.py:1098-1100): they go to the next pool; false when it is full
template <class T, class E>
__device__ bool bw_jw_carry(const T& t, const E& e, const JwPool& pool, const u32* perm, u32 qb, u32 qe, bool woken, u64 s, u32 keep,
                            JwState& st) {
  const u64 b = atomicAdd(e.n_next, (unsigned long long)keep);
  if (b + keep > e.max_queue) {
    bw_jw_fail(t, BW_JW_FULL_QUEUE);
    return false;
  }
  u64 w = b;
  for (u32 i = qb; i < qe; ++i) {
    const u32 x = perm[i];
    if (pool.side[x] == BW_JW_DROP || (woken && pool.ts[x] <= st.wm)) continue;
    if (w == b) st.q0ts = pool.ts[x];
    e.next.slot[w] = (u32)s;
    e.next.ts[w] = pool.ts[x];
    e.next.h[w] = pool.h[x];
    e.next.side[w] = pool.side[x];
    ++w;
  }
  return true;
}

// pass B, one thread per slot: a woken key plays its due entries (already in ts order, ties in arrival order), keeps
// the others queued in arrival order, and closes; an idle key's entries move to the next pool unchanged
__global__ void k_jwin_flush(JwTable t, JwEmit e, JwParams p, JwPool pool, const u32* perm) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    JwState st = t.st[s];
    if (!st.init) continue;
    const bool woken = st.act == p.ord;
    const u32 qb = st.qord == p.ord ? st.qb : 0, qe = st.qord == p.ord ? st.qe : 0;
    if (!woken && qb == qe) continue;
    const u64 key = t.keys[s];
    JwWin* W = t.win + s * (u64)t.M;
    u64 seq = 0, mseq = 0;
    u32 nw = st.n, keep = 0;
    bool full = false;
    for (u32 i = qb; i < qe; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] == BW_JW_DROP) continue;
      if (woken && pool.ts[x] <= st.wm) {
        if (!full) full = !bw_jw_play(t, e, p, key, W, nw, pool.ts[x], pool.h[x], pool.side[x], seq);
      } else {
        ++keep;
      }
    }
    if (full) {
      bw_jw_fail(t, BW_JW_FULL_WINDOWS);
      continue;
    }
    if (keep && !bw_jw_carry(t, e, pool, perm, qb, qe, woken, s, keep, st)) continue;
    st.nq = keep;
    if (woken) {
      bw_jw_close_windows(t, e, p, key, W, nw, st.wm, seq, mseq);
      st.n = nw;
      if (nw == 0 && keep == 0) st.init = 0;  // discarded with its clock (windowing.py:1110-1113)
    }
    t.st[s] = st;
  }
}

__global__ void k_jwin_init(JwTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.keys[s] = BW_EMPTY_KEY;
    t.st[s].init = 0;
    t.st[s].n = t.st[s].nq = 0;
    t.st[s].qord = ~0ULL;
    t.st[s].act = ~0ULL;
  }
}
