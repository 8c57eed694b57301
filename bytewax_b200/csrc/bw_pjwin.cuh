// bw_pjwin.cuh -- K14: `join_window` with insert mode product over tumbling and sliding windows.
//
// The reference runs `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) over
// `_SlidingWindowerLogic` (:603-668) with one `_JoinWindowLogic` (:1849-1902) per window whose `_JoinState`
// (operators/__init__.py:2072-2120) keeps one list per side: `add_val` appends, `astuples` is the `itertools.product` of
// the lists (an empty side gives one None), `clear` empties every list.  "complete" emits the product and clears once
// every side is non-empty; "running" emits it after every value; "final" at the close.
//
// The per-key steps are K8's (bw_jwin.cuh), called, not restated: the activation is grouped by key, one thread per key
// runs the late test; unordered, the same thread plays the on-time values and closes (k_pjwin_apply); ordered, the
// values join K8's pool, K8's sort kernels put it in play order, and one thread per slot plays, carries over and closes
// (k_pjwin_flush); notify and EOF mark the keys with K8's k_jwin_mark.
//
// A window's lists are K9's ENTRY STORE (bw_collect.cuh) with the side in the reference word: one entry per (played
// value, window) -- the window's cell and the side, the value's rank within (window, side), the handle.  Per window and
// side the thread keeps the value count and the first rank of the current generation (a "complete" clear moves it up to
// the count), so the lists are always the ranks [gen, cnt).  An emission only appends an EVENT: key, window, epoch,
// call, sequence and per side a rank range [lo, hi).  Every window that emits in a call gets one STAGE RECORD covering
// the union of its events' ranges, and after the per-key kernels k_pjwin_gather copies those entries, over the whole
// store, into staging -- so each event can still be expanded at advance, after later calls compacted the store.
//
// At advance / eof the events are put in the reference's order (order_perm: per call, ascending key string, then play
// order), each event's row count is prod_s max(1, hi_s - lo_s), and k_pjwin_expand writes one output row per thread:
// it finds its event by binary search over the exclusive scan of the counts and decodes the mixed radix with the last
// side varying fastest (`itertools.product`).
//
// Releases: an entry dies when its window closes or a "complete" clear passes its rank; a value's handle is released
// when its last entry dies (a per-value live-entry count, set at play), in the call in which that happens.  K9's rule
// -- the entry of the highest window id releases -- does not hold here: in "complete" mode a sliding window can clear
// a value a lower window still holds.
//
// Per key:
//   keys[slot], st[slot]   as K8 (JwTable; its JwWin array is not used)
//   win[slot * M ...]      open windows in first-opened order: id, cell
//   cell[slot * M + cell]  per side the value count and the generation's first rank
//   rec_ord / rec_c        [slot * M + cell]: the call in which the window on that cell last got a stage record, and it
//   close_ord              [slot * M + cell]: the call in which the window on that cell closed
#pragma once
#include "../../include/bwgpu.h"
#include "bw_common.cuh"
#include "bw_jwin.cuh"
#include "bw_collect.cuh"

// reasons behind a BW_ERR_CAPACITY beyond K8's and K9's, or-ed into JwTable::why
enum { BW_PJ_FULL_SIDE = 128 };  // a side list of one window reached 2^32 values

struct PjWin {
  i64 id;
  u32 cell;
  u32 pad;
  __device__ void open(i64 i) { id = i; }
};
struct PjCell {
  u32 cnt[BW_JW_MAXSIDES];  // values played into the window, per side
  u32 gen[BW_JW_MAXSIDES];  // rank of the first value of the side's current list
};
struct PjTable {
  JwTable j;  // keys, clock / queue state, error words, cap, M, sides
  PjWin* win;
  PjCell* cell;
  u64* rec_ord;
  u64* rec_c;
  u64* close_ord;
  // the fail / release helpers of bw_jwin.cuh read these two
  u32* err;
  u32* why;
};
struct PjStore {
  CwStore c;    // ref = ((slot * M + cell) << 2) | side, or BW_CW_DEAD; rank within (window, side); handle
  u64* vi;      // the entry's value
  u32* vcnt;    // [value]: its live entries; the decrement to zero releases the handle
  u64 vcap;
  unsigned long long* nv;
  unsigned long long* n_dead;  // entries that died in this call
};
struct PjEmit {
  // emission events
  u64 *key, *wid, *epoch, *ord, *seq, *rec;
  u32 *lo, *hi;  // [event * 4 + side]: the side's list is ranks [lo, hi) of the window
  u64 max_rows;
  unsigned long long* n_rows;
  // meta: closed windows
  u64 *m_key, *m_wid, *m_epoch, *m_ord, *m_seq;
  unsigned long long* n_meta;
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
  // stage records, one per (window, call) with events: per side the first rank b and the count n staged, and where
  // they start in staging
  u32 *rb, *rn;  // [record * 4 + side]
  u64* rbase;    // [record * 4 + side]
  unsigned long long* n_rec;  // (records <= events: bounded by max_rows)
  u64* stage;
  u64 max_stage;
  unsigned long long* n_stage;
};

// reserve `entries` entries and `vals` values of the store for one key; false (and the call fails) when they do not fit
__device__ __forceinline__ bool bw_pj_reserve(const PjTable& t, const PjStore& es, u64 entries, u64 vals, u64& ei, u64& vi) {
  ei = entries ? atomicAdd(es.c.n, (unsigned long long)entries) : 0;
  vi = vals ? atomicAdd(es.nv, (unsigned long long)vals) : 0;
  if (ei + entries <= es.c.cap && vi + vals <= es.vcap) return true;
  bw_jw_fail(t, BW_CW_FULL_STORE);
  return false;
}

// one emission of the window w: an event naming per side the ranks [gen, cnt), and the window's stage record of this
// call (opened on its first event, with the ranks it starts at; each event extends it to its hi)
__device__ void bw_pj_emit(const PjTable& t, const PjEmit& e, const JwParams& p, u64 key, u64 slot, const PjWin& w, u64& seq,
                           u64& touched) {
  const u64 cell = slot * (u64)t.j.M + w.cell;
  const PjCell c = t.cell[cell];
  const int sides = t.j.sides;
  u64 r = t.rec_c[cell];
  if (t.rec_ord[cell] != p.ord) {
    r = atomicAdd(e.n_rec, 1ULL);
    if (r >= e.max_rows) {
      bw_jw_fail(t, BW_JW_FULL_EMIT);
      return;
    }
    for (int s = 0; s < BW_JW_MAXSIDES; ++s) {
      e.rb[r * 4 + s] = s < sides ? c.gen[s] : 0;
      e.rn[r * 4 + s] = 0;
    }
    t.rec_ord[cell] = p.ord;
    t.rec_c[cell] = r;
    touched |= 1ULL << w.cell;
  }
  const u64 row = atomicAdd(e.n_rows, 1ULL);
  if (row >= e.max_rows) {
    bw_jw_fail(t, BW_JW_FULL_EMIT);
    return;
  }
  e.key[row] = key;
  e.wid[row] = (u64)w.id;
  e.epoch[row] = p.epoch;
  e.ord[row] = p.ord;
  e.seq[row] = seq++;
  e.rec[row] = r;
  for (int s = 0; s < BW_JW_MAXSIDES; ++s) {
    const bool on = s < sides;
    e.lo[row * 4 + s] = on ? c.gen[s] : 0;
    e.hi[row * 4 + s] = on ? c.cnt[s] : 0;
    if (on) e.rn[r * 4 + s] = c.cnt[s] - e.rb[r * 4 + s];
  }
}

// one due value: `_handle_inserts` (windowing.py:1064-1077) -- `add_val` in every window of open_for(ts), ascending id,
// as the entries at es[ei...] of value v, then `_JoinWindowLogic.on_value` (:1866-1876); 0, or the BW_* reason the key
// cannot go on
__device__ u32 bw_pj_play(const PjTable& t, const PjEmit& e, const PjStore& es, const JwParams& p, u64 key, u64 slot, PjWin* W, u32& n,
                          i64 ts, u64 h, int side, u64 v, u64& ei, u64& seq, u64& touched) {
  const u32 M = (u32)t.j.M;
  const int sides = t.j.sides;
  i64 lo, hi;
  bw_jw_ids(p, ts, lo, hi);
  es.vcnt[v] = (u32)(hi - lo + 1);  // (at most M: more fails below)
  for (i64 id = lo; id <= hi; ++id) {
    const u32 n0 = n;
    const u32 i = bw_jw_find_or_open(W, n, M, id);
    if (i == M) return BW_JW_FULL_WINDOWS;
    const u64 base = slot * M;
    if (n > n0) {  // a new window: the lowest cell no open window of the key has, with empty lists
      u64 used = 0;
      for (u32 k = 0; k < n0; ++k) used |= 1ULL << W[k].cell;
      W[i].cell = (u32)__ffsll((long long)~used) - 1;
      t.cell[base + W[i].cell] = PjCell{};
    }
    const u64 cell = base + W[i].cell;
    PjCell& c = t.cell[cell];
    if (c.cnt[side] == 0xFFFFFFFFu) return BW_PJ_FULL_SIDE;
    es.c.ref[ei] = (cell << 2) | (u64)side;
    es.c.rank[ei] = c.cnt[side]++;
    es.c.h[ei] = h;
    es.vi[ei] = v;
    ++ei;
    if (p.emit_mode == BW_JOIN_EMIT_COMPLETE) {
      bool all = true;
      for (int s = 0; s < sides; ++s) all = all && c.cnt[s] > c.gen[s];
      if (all) {
        bw_pj_emit(t, e, p, key, slot, W[i], seq, touched);
        for (int s = 0; s < sides; ++s) c.gen[s] = c.cnt[s];  // _JoinState.clear
      }
    } else if (p.emit_mode == BW_JOIN_EMIT_RUNNING) {
      bw_pj_emit(t, e, p, key, slot, W[i], seq, touched);
    }
  }
  return 0;
}

// `_handle_closed` (windowing.py:1087-1093): windows with close <= watermark in first-opened order; `final` event, then
// the meta row; every entry of a closed window dies in this call's gather
__device__ void bw_pj_close(const PjTable& t, const PjEmit& e, const JwParams& p, u64 key, u64 slot, PjWin* W, u32& n, i64 wm, u64& seq,
                            u64& touched) {
  u64 mseq = 0;
  bw_jw_close_each(p, W, n, wm, [&](const PjWin& w) {
    if (p.emit_mode == BW_JOIN_EMIT_FINAL) bw_pj_emit(t, e, p, key, slot, w, seq, touched);
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
    t.close_ord[slot * (u64)t.j.M + w.cell] = p.ord;
  });
}

// the key's stage records of this call (cells in `touched`) each reserve their staging range, side after side
__device__ void bw_pj_stage(const PjTable& t, const PjEmit& e, u64 slot, u64 touched) {
  while (touched) {
    const int c = __ffsll((long long)touched) - 1;
    touched &= touched - 1;
    const u64 r = t.rec_c[slot * (u64)t.j.M + c];
    u64 tot = 0;
    for (int s = 0; s < BW_JW_MAXSIDES; ++s) tot += e.rn[r * 4 + s];
    u64 at = atomicAdd(e.n_stage, (unsigned long long)tot);
    if (at + tot > e.max_stage) {  // (sized by the host for every entry held: never reached)
      bw_jw_fail(t, BW_CW_FULL_STORE);
      return;
    }
    for (int s = 0; s < BW_JW_MAXSIDES; ++s) {
      e.rbase[r * 4 + s] = at;
      at += e.rn[r * 4 + s];
    }
  }
}

// pass A, one thread per key segment: K8's late test per item; unordered, then the play of the on-time items in arrival
// order and the close; ordered, the on-time items go to the pool at base + q
__global__ void k_pjwin_apply(PjTable t, PjEmit e, PjStore es, JwParams p, JwPool pool, u64 base, const u64* ksorted, const u32* isorted,
                              const u32* headpos, const u64* handles, const unsigned char* sides, const i64* ts_us, unsigned char* late,
                              u64 n) {
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
    u64 lseq = 0, entries = 0, vals = 0;
    for (u64 q = h; q < end; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      if (sides[o] >= t.j.sides) {  // (device columns are not checked on the host)
        bw_jw_bad_side(t.j);
        if (p.ordered) {
          pool.slot[base + q] = (u32)s;
          pool.side[base + q] = (unsigned char)BW_JW_DROP;
        } else {
          late[q] = 1;
        }
        continue;
      }
      const bool is_late = bw_jw_on_item(st, p, ts, wm);
      if (is_late) {
        bw_jw_late_rows(t, e, p, key, ts, o, lseq);
        bw_jw_release(t, e, handles[o]);
      } else {
        entries += bw_cw_nwin(p, ts);
        ++vals;
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
      u64 ei, vi;
      if (!bw_pj_reserve(t, es, entries, vals, ei, vi)) continue;
      const u64 eend = ei + entries;
      PjWin* W = t.win + s * (u64)t.j.M;
      u32 nw = st.n, bad = 0;
      u64 seq = 0, touched = 0;
      for (u64 q = h; q < end && !bad; ++q) {
        if (late[q]) continue;
        const u32 o = isorted[q];
        bad = bw_pj_play(t, e, es, p, key, s, W, nw, ts_us[o], handles[o], sides[o], vi++, ei, seq, touched);
      }
      if (bad) {
        bw_cw_kill(es.c, ei, eend);
        bw_jw_fail(t, bad);
        continue;  // the call fails and the join refuses further work
      }
      bw_pj_close(t, e, p, key, s, W, nw, wm, seq, touched);
      bw_pj_stage(t, e, s, touched);
      st.n = nw;
      if (nw == 0) st.init = 0;  // _is_empty (windowing.py:1110-1113): the engine discards the logic, clock included
    }
    t.j.st[s] = st;
  }
}

// pass B (ordered, notify, EOF), one thread per slot: a woken key plays its due entries (already in ts order, ties in
// arrival order), keeps the others queued, and closes; an idle key's entries move to the next pool unchanged
__global__ void k_pjwin_flush(PjTable t, PjEmit e, PjStore es, JwParams p, JwPool pool, const u32* perm) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.j.cap; s += (u64)gridDim.x * blockDim.x) {
    JwState st = t.j.st[s];
    if (!st.init) continue;
    const bool woken = st.act == p.ord;
    const u32 qb = st.qord == p.ord ? st.qb : 0, qe = st.qord == p.ord ? st.qe : 0;
    if (!woken && qb == qe) continue;
    u32 keep = 0;
    u64 entries = 0, vals = 0;
    for (u32 i = qb; i < qe; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] == BW_JW_DROP) continue;
      if (woken && pool.ts[x] <= st.wm) {
        entries += bw_cw_nwin(p, pool.ts[x]);
        ++vals;
      } else {
        ++keep;
      }
    }
    u64 ei, vi;
    if (!bw_pj_reserve(t, es, entries, vals, ei, vi)) continue;
    const u64 eend = ei + entries;
    const u64 key = t.j.keys[s];
    PjWin* W = t.win + s * (u64)t.j.M;
    u32 nw = st.n, bad = 0;
    u64 seq = 0, touched = 0;
    for (u32 i = qb; i < qe && !bad; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] != BW_JW_DROP && woken && pool.ts[x] <= st.wm)
        bad = bw_pj_play(t, e, es, p, key, s, W, nw, pool.ts[x], pool.h[x], pool.side[x], vi++, ei, seq, touched);
    }
    if (bad) {
      bw_cw_kill(es.c, ei, eend);
      bw_jw_fail(t, bad);
      continue;
    }
    if (keep && !bw_jw_carry(t, e, pool, perm, qb, qe, woken, s, keep, st)) continue;
    st.nq = keep;
    if (woken) {
      bw_pj_close(t, e, p, key, s, W, nw, st.wm, seq, touched);
      bw_pj_stage(t, e, s, touched);
      st.n = nw;
      if (nw == 0 && keep == 0) st.init = 0;  // discarded with its clock (windowing.py:1110-1113)
    }
    t.j.st[s] = st;
  }
}

// after the per-key kernels of a call, over the whole store: an entry inside its window's stage record of this call is
// copied to staging (the window may stay open); an entry whose window closed in this call, or whose rank a clear passed,
// dies, and the death of a value's last entry releases its handle.  Nothing to do when the call made no record and
// closed no window (rec0, meta0: the counts before the call), nor after a failed call (records may lack staging).
__global__ void k_pjwin_gather(PjTable t, PjEmit e, PjStore es, JwParams p, u64 rec0, u64 meta0) {
  if (*t.err) return;
  if (*e.n_rec == rec0 && *e.n_meta == meta0) return;
  const u64 n = *es.c.n;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  for (u64 b = (u64)blockIdx.x * blockDim.x; b < n; b += stride) {  // (b is warp-uniform: the whole warp reaches the ballots)
    const u64 i = b + threadIdx.x;
    bool dead = false, rel = false;
    u64 h = 0;
    if (i < n) {
      const u64 r = es.c.ref[i];
      if (r != BW_CW_DEAD) {
        const u64 cell = r >> 2;
        const int s = (int)(r & 3);
        const u32 rank = es.c.rank[i];
        h = es.c.h[i];
        if (t.rec_ord[cell] == p.ord) {
          const u64 c = t.rec_c[cell];
          const u32 d = rank - e.rb[c * 4 + s];  // (wraps above every count when rank < b)
          if (d < e.rn[c * 4 + s]) e.stage[e.rbase[c * 4 + s] + d] = h;
        }
        if (t.close_ord[cell] == p.ord || rank < t.cell[cell].gen[s]) {
          dead = true;
          es.c.ref[i] = BW_CW_DEAD;
          rel = atomicSub(&es.vcnt[es.vi[i]], 1u) == 1u;
        }
      }
    }
    const unsigned md = __ballot_sync(0xffffffffu, dead);
    if (lane == 0 && md) atomicAdd(es.n_dead, (unsigned long long)__popc(md));
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

// value compaction: 1 for a value with live entries (u64, for the scan that maps old value indices to new ones)
__global__ void k_pjwin_vlive(const u32* vcnt, u64* live, unsigned char* flag, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    live[i] = vcnt[i] != 0;
    flag[i] = vcnt[i] != 0;
  }
}
// after both compactions: every live entry's value index through the scan of the value flags
__global__ void k_pjwin_remap(u64* vi, const u64* vmap, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) vi[i] = vmap[vi[i]];
}

// a + b, saturating at 2^64 - 1 (the scan of the row counts)
struct PjSatAdd {
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const {
    const u64 s = a + b;
    return s < a ? ~0ULL : s;
  }
};

// the expansion's view of the events in the reference's order
struct PjOrdered {
  u64 *cnt, *key, *wid, *epoch;
  u64* base;  // [side * n + i]: where event i's list of that side starts in staging
  u32* len;   // [side * n + i]: its length (0: the side contributes one None)
};

// advance / eof: event perm[i] is the i-th in the reference's order: its row count prod max(1, len) (saturating), its
// columns, and per side its list in staging
__global__ void k_pjwin_count(PjEmit e, PjOrdered o, int sides, const u32* perm, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const u32 x = perm[i];
    const u64 r = e.rec[x];
    u64 c = 1;
    for (int s = 0; s < sides; ++s) {
      const u32 lo = e.lo[(u64)x * 4 + s], len = e.hi[(u64)x * 4 + s] - lo;
      o.base[s * n + i] = e.rbase[r * 4 + s] + (lo - e.rb[r * 4 + s]);
      o.len[s * n + i] = len;
      if (len > 1) c = c > ~0ULL / len ? ~0ULL : c * len;
    }
    o.cnt[i] = c;
    o.key[i] = e.key[x];
    o.wid[i] = e.wid[x];
    o.epoch[i] = e.epoch[x];
  }
}

struct PjRows {  // the output columns (bw_jwin_rows)
  u64 *key, *wid, *h0, *h1, *h2, *h3, *mask, *epoch;
};

// one output row per thread, grid-stride, in order: its event is the last one whose offset is <= the row (every event
// has at least one row); row q of the event takes index (q / prod_{t>s} n_t) % n_s on side s
__global__ void k_pjwin_expand(PjOrdered o, const u64* off, u64 nev, int sides, const u64* stage, PjRows out, u64 total) {
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < total; r += (u64)gridDim.x * blockDim.x) {
    u64 lo = 0, hi = nev;  // off[lo] <= r < off[hi]
    while (hi - lo > 1) {
      const u64 mid = lo + (hi - lo) / 2;
      if (off[mid] <= r) lo = mid;
      else hi = mid;
    }
    u64 q = r - off[lo], mask = 0;
    u64 hs[BW_JW_MAXSIDES] = {0, 0, 0, 0};
#pragma unroll
    for (int s = BW_JW_MAXSIDES - 1; s >= 0; --s) {
      if (s >= sides) continue;
      const u32 len = o.len[s * nev + lo];
      if (!len) continue;
      u64 idx;
      if (q >> 32) {
        idx = q % len;
        q /= len;
      } else {
        idx = (u32)q % len;
        q = (u32)q / len;
      }
      hs[s] = stage[o.base[s * nev + lo] + idx];
      mask |= 1ULL << s;
    }
    out.key[r] = o.key[lo];
    out.wid[r] = o.wid[lo];
    out.h0[r] = hs[0];
    out.h1[r] = hs[1];
    out.h2[r] = hs[2];
    out.h3[r] = hs[3];
    out.mask[r] = mask;
    out.epoch[r] = o.epoch[lo];
  }
}

__global__ void k_pjwin_init(PjTable t) {
  const u64 cells = (t.j.cap + 1) * (u64)t.j.M;
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < cells; s += (u64)gridDim.x * blockDim.x) {
    t.rec_ord[s] = ~0ULL;
    t.close_ord[s] = ~0ULL;
    if (s > t.j.cap) continue;
    t.j.keys[s] = BW_EMPTY_KEY;
    t.j.st[s].init = 0;
    t.j.st[s].n = t.j.st[s].nq = 0;
    t.j.st[s].qord = ~0ULL;
    t.j.st[s].act = ~0ULL;
  }
}
