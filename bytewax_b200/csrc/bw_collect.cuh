// bw_collect.cuh -- K9: `collect_window` into list / set / dict over tumbling and sliding windows.
//
// The reference runs `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) over
// `_SlidingWindowerLogic` (:603-668) with one `_FoldWindowLogic` (:1046-1190) per window whose folder appends, adds or
// sets each value (`_collect_get_callbacks`, :1356-1384).  The window's state is its values in play order, so the
// device keeps exactly that, as handles: every (played value, window) pair is one entry of an ENTRY STORE -- the
// window, the value's rank in it, the handle -- and the host builds the container from the window's handles.
//
// The per-key steps are K8's (bw_jwin.cuh), called, not restated: the activation is grouped by key, one thread per key
// runs the late test (bw_jw_on_item, bw_jw_late_rows); unordered, the same thread plays the on-time values and closes
// (k_cwin_apply); ordered, the values join K8's pool, which K8's sort kernels put in play order, and one thread per slot
// plays the due entries, carries the rest over (bw_jw_carry) and closes (k_cwin_flush); notify and EOF mark the keys
// with K8's k_jwin_mark.  Playing a value only appends entries: the thread never copies a window's list.
//
// The close gives each closing window a record (key, id, value count) and a range of a staging buffer reserved by its
// count; then k_cwin_gather, over the whole store, moves every entry of a window that closed in this call to
// `range start + rank`, so a window of 10^6 values is materialised by the whole grid.  The entry is then dead; dead
// entries leave the store by stream compaction once they outnumber the live ones (host side).  At advance / eof the
// records are put in the reference's order and the staging ranges copied to the output in that order (host side).
//
// Handles: a value's windows close in id order (a key's windows close by `close <= watermark`, and close grows with
// the id), so its handle is released by the entry of its highest window id, in the call that closes that window; a
// late item's handle in the call that received it.
//
// Per key:
//   keys[slot], st[slot]   as K8 (JwTable; its JwWin array is not used)
//   win[slot * M ...]      open windows in first-opened order: id, value count, cell
//   cell_ord / cell_c      [slot * M + cell]: the call in which the window on that cell last closed, and its record
// A window's cell is a number in [0, M) no other open window of the key has; entries name (slot * M + cell), which
// stays put while the first-opened list shifts.
#pragma once
#include "../../include/bwgpu.h"
#include "bw_common.cuh"
#include "bw_jwin.cuh"

#define BW_CW_DEAD (~0ULL)  // an entry already moved out (its window closed)
enum { BW_CW_FULL_STORE = 64 };  // (the host sizes the store for every entry a call can add: never reached)

struct CwWin {
  i64 id;
  u32 cnt;   // values played into the window
  u32 cell;
  __device__ void open(i64 i) {
    id = i;
    cnt = 0;
  }
};
struct CwTable {
  JwTable j;  // keys, clock / queue state, error words, cap, M
  CwWin* win;
  u64* cell_ord;
  u64* cell_c;
  // the fail / release helpers of bw_jwin.cuh read these two
  u32* err;
  u32* why;
};
struct CwStore {  // one entry per (played value, window)
  u64* ref;       // ((slot * M + cell) << 1) | (window is the value's highest id), or BW_CW_DEAD
  u32* rank;      // position of the value in its window's list
  u64* h;
  u64 cap;
  unsigned long long* n;
};
struct CwEmit {
  // closed windows: one record each (the `E` row and its `M` row)
  u64 *key, *wid, *cnt, *soff, *epoch, *ord, *seq;
  u64 max_rows;
  unsigned long long* n_rows;
  // late items, one row per window id (names as JwEmit: bw_jw_late_rows)
  u64 *l_key, *l_wid, *l_epoch, *l_act, *l_row, *l_ord, *l_seq;
  u64 max_late;
  unsigned long long* n_late;
  // released handles
  u64* rel;
  u64 max_rel;
  unsigned long long* n_rel;
  // ordered mode: entries carried over to the next pool (bw_jw_carry)
  JwPool next;
  u64 max_queue;
  unsigned long long* n_next;
  // staging: the handles of the closed windows, record c's at [soff[c], soff[c] + cnt[c]); stage_rec names the record
  u64* stage;
  u32* stage_rec;
  u64 max_stage;
  unsigned long long* n_stage;
};

__device__ __forceinline__ u64 bw_cw_nwin(const JwParams& p, i64 ts) {
  i64 lo, hi;
  bw_jw_ids(p, ts, lo, hi);
  return hi >= lo ? (u64)(hi - lo + 1) : 0;
}

// reserve n entries of the store for one key; false (and the call fails) when they do not fit
__device__ __forceinline__ bool bw_cw_reserve(const CwTable& t, const CwStore& es, u64 n, u64& at) {
  at = n ? atomicAdd(es.n, (unsigned long long)n) : 0;
  if (at + n <= es.cap) return true;
  bw_jw_fail(t, BW_CW_FULL_STORE);
  return false;
}

// one due value: `_handle_inserts` (windowing.py:1064-1077) -- it joins every window of open_for(ts), ascending id, as
// the entries at es[ei...]; false when the key needs more than M windows
__device__ bool bw_cw_play(const CwTable& t, const CwStore& es, const JwParams& p, u64 slot, CwWin* W, u32& n, i64 ts, u64 h, u64& ei) {
  const u32 M = (u32)t.j.M;
  i64 lo, hi;
  bw_jw_ids(p, ts, lo, hi);
  for (i64 id = lo; id <= hi; ++id) {
    const u32 n0 = n;
    const u32 i = bw_jw_find_or_open(W, n, M, id);
    if (i == M) return false;
    if (n > n0) {  // a new window: the lowest cell no open window of the key has
      u64 used = 0;
      for (u32 k = 0; k < n0; ++k) used |= 1ULL << W[k].cell;
      W[i].cell = (u32)__ffsll((long long)~used) - 1;
    }
    es.ref[ei] = ((slot * M + W[i].cell) << 1) | (id == hi ? 1ULL : 0ULL);
    es.rank[ei] = W[i].cnt++;
    es.h[ei] = h;
    ++ei;
  }
  return true;
}

// the key's closing windows, first-opened order: a record each, and a staging range for k_cwin_gather
__device__ void bw_cw_close(const CwTable& t, const CwEmit& e, const JwParams& p, u64 key, u64 slot, CwWin* W, u32& n, i64 wm) {
  u64 seq = 0;
  bw_jw_close_each(p, W, n, wm, [&](const CwWin& w) {
    const u64 c = atomicAdd(e.n_rows, 1ULL);
    if (c >= e.max_rows) {
      bw_jw_fail(t, BW_JW_FULL_EMIT);
      return;
    }
    const u64 at = atomicAdd(e.n_stage, (unsigned long long)w.cnt);
    if (at + w.cnt > e.max_stage) {  // (sized by the host for every entry held: never reached)
      bw_jw_fail(t, BW_CW_FULL_STORE);
      return;
    }
    e.key[c] = key;
    e.wid[c] = (u64)w.id;
    e.cnt[c] = w.cnt;
    e.soff[c] = at;
    e.epoch[c] = p.epoch;
    e.ord[c] = p.ord;
    e.seq[c] = seq++;
    const u64 cell = slot * (u64)t.j.M + w.cell;
    t.cell_c[cell] = c;
    t.cell_ord[cell] = p.ord;
  });
}

// the entries [ei, end) a failed key reserved and did not write: dead, so k_cwin_gather skips them
__device__ __forceinline__ void bw_cw_kill(const CwStore& es, u64 ei, u64 end) {
  for (; ei < end; ++ei) es.ref[ei] = BW_CW_DEAD;
}

// pass A, one thread per key segment: K8's late test per item; unordered, then the play of the on-time items in arrival
// order and the close; ordered, the on-time items go to the pool at base + q
__global__ void k_cwin_apply(CwTable t, CwEmit e, CwStore es, JwParams p, JwPool pool, u64 base, const u64* ksorted, const u32* isorted,
                             const u32* headpos, const u64* handles, const i64* ts_us, unsigned char* late, u64 n) {
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.j.keys, t.j.cap, key, t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      for (u64 q = h; q < n && ksorted[q] == key; ++q)  // (the pool sort and flush still read these entries)
        if (p.ordered) {
          pool.slot[base + q] = (u32)t.j.cap;
          pool.side[base + q] = (unsigned char)BW_JW_DROP;
        }
      continue;
    }
    JwState st = t.j.st[s];
    bw_jw_begin(st, p);
    u64 end = h;
    while (end < n && ksorted[end] == key) ++end;
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0, entries = 0;
    for (u64 q = h; q < end; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      const bool is_late = bw_jw_on_item(st, p, ts, wm);
      if (is_late) {
        bw_jw_late_rows(t, e, p, key, ts, o, lseq);
        bw_jw_release(t, e, handles[o]);
      } else {
        entries += bw_cw_nwin(p, ts);
      }
      if (p.ordered) {
        pool.slot[base + q] = (u32)s;
        pool.ts[base + q] = ts;
        pool.h[base + q] = handles[o];
        pool.side[base + q] = is_late ? (unsigned char)BW_JW_DROP : 0;
      } else {
        late[q] = is_late;
      }
    }
    st.wm = wm;
    st.act = p.ord;
    if (!p.ordered) {  // every queued entry is due, in arrival order
      u64 ei;
      if (!bw_cw_reserve(t, es, entries, ei)) continue;
      const u64 eend = ei + entries;
      CwWin* W = t.win + s * (u64)t.j.M;
      u32 nw = st.n;
      bool full = false;
      for (u64 q = h; q < end && !full; ++q) {
        if (late[q]) continue;
        const u32 o = isorted[q];
        full = !bw_cw_play(t, es, p, s, W, nw, ts_us[o], handles[o], ei);
      }
      if (full) {
        bw_cw_kill(es, ei, eend);
        bw_jw_fail(t, BW_JW_FULL_WINDOWS);
        continue;  // the call fails and the collect refuses further work
      }
      bw_cw_close(t, e, p, key, s, W, nw, wm);
      st.n = nw;
      if (nw == 0) st.init = 0;  // _is_empty (windowing.py:1110-1113): the engine discards the logic, clock included
    }
    t.j.st[s] = st;
  }
}

// pass B (ordered, notify, EOF), one thread per slot: a woken key plays its due entries (already in ts order, ties in
// arrival order), keeps the others queued, and closes; an idle key's entries move to the next pool unchanged
__global__ void k_cwin_flush(CwTable t, CwEmit e, CwStore es, JwParams p, JwPool pool, const u32* perm) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.j.cap; s += (u64)gridDim.x * blockDim.x) {
    JwState st = t.j.st[s];
    if (!st.init) continue;
    const bool woken = st.act == p.ord;
    const u32 qb = st.qord == p.ord ? st.qb : 0, qe = st.qord == p.ord ? st.qe : 0;
    if (!woken && qb == qe) continue;
    u32 keep = 0;
    u64 entries = 0;
    for (u32 i = qb; i < qe; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] == BW_JW_DROP) continue;
      if (woken && pool.ts[x] <= st.wm) entries += bw_cw_nwin(p, pool.ts[x]);
      else ++keep;
    }
    u64 ei;
    if (!bw_cw_reserve(t, es, entries, ei)) continue;
    const u64 eend = ei + entries;
    CwWin* W = t.win + s * (u64)t.j.M;
    u32 nw = st.n;
    bool full = false;
    for (u32 i = qb; i < qe && !full; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] != BW_JW_DROP && woken && pool.ts[x] <= st.wm) full = !bw_cw_play(t, es, p, s, W, nw, pool.ts[x], pool.h[x], ei);
    }
    if (full) {
      bw_cw_kill(es, ei, eend);
      bw_jw_fail(t, BW_JW_FULL_WINDOWS);
      continue;
    }
    if (keep && !bw_jw_carry(t, e, pool, perm, qb, qe, woken, s, keep, st)) continue;
    st.nq = keep;
    if (woken) {
      bw_cw_close(t, e, p, t.j.keys[s], s, W, nw, st.wm);
      st.n = nw;
      if (nw == 0 && keep == 0) st.init = 0;  // discarded with its clock (windowing.py:1110-1113)
    }
    t.j.st[s] = st;
  }
}

// every entry of a window that closed in this call goes to its record's staging range at its rank, and is dead; the
// entry of a value's highest window releases the handle.  Nothing to do when the call closed no window (rows0: the
// record count before the call).
__global__ void k_cwin_gather(CwTable t, CwEmit e, CwStore es, JwParams p, u64 rows0) {
  if (*e.n_rows == rows0) return;
  const u64 n = *es.n;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  for (u64 b = (u64)blockIdx.x * blockDim.x; b < n; b += stride) {  // (b is warp-uniform: the whole warp reaches the ballot)
    const u64 i = b + threadIdx.x;
    bool rel = false;
    u64 h = 0;
    if (i < n) {
      const u64 r = es.ref[i];
      if (r != BW_CW_DEAD && t.cell_ord[r >> 1] == p.ord) {
        const u64 c = t.cell_c[r >> 1];
        const u64 j = e.soff[c] + es.rank[i];
        h = es.h[i];
        e.stage[j] = h;
        e.stage_rec[j] = (u32)c;
        es.ref[i] = BW_CW_DEAD;
        rel = r & 1;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, rel);
    if (!m) continue;
    u64 at = 0;
    if (lane == (unsigned)__ffs(m) - 1) at = atomicAdd(e.n_rel, (unsigned long long)__popc(m));
    at = __shfl_sync(0xffffffffu, at, __ffs(m) - 1) + __popc(m & ((1u << lane) - 1));
    if (rel) {
      if (at < e.max_rel) e.rel[at] = h;  // (sized by the host for every handle the call can release: never reached)
      else bw_jw_fail(t, BW_JW_FULL_EMIT);
    }
  }
}

// compaction flags: 1 for a live entry
__global__ void k_cwin_live(const u64* ref, unsigned char* flag, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) flag[i] = ref[i] != BW_CW_DEAD;
}

// advance / eof: record perm[i] is the i-th in the reference's order; inv[perm[i]] = i and its count in that order
__global__ void k_cwin_order(const u32* perm, const u64* cnt, u32* inv, u64* cnt_sorted, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    inv[perm[i]] = (u32)i;
    cnt_sorted[i] = cnt[perm[i]];
  }
}
// every staged handle to its place in the output: record c's list starts at off[inv[c]]
__global__ void k_cwin_place(const u64* stage, const u32* stage_rec, const u64* soff, const u32* inv, const u64* off, u64* out, u64 n) {
  for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (u64)gridDim.x * blockDim.x) {
    const u32 c = stage_rec[j];
    out[off[inv[c]] + (j - soff[c])] = stage[j];
  }
}

__global__ void k_cwin_init(CwTable t) {
  const u64 cells = (t.j.cap + 1) * (u64)t.j.M;
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < cells; s += (u64)gridDim.x * blockDim.x) {
    t.cell_ord[s] = ~0ULL;
    if (s > t.j.cap) continue;
    t.j.keys[s] = BW_EMPTY_KEY;
    t.j.st[s].init = 0;
    t.j.st[s].n = t.j.st[s].nq = 0;
    t.j.st[s].qord = ~0ULL;
    t.j.st[s].act = ~0ULL;
  }
}
