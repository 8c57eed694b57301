// bw_argwin.cuh -- K11: `max_window` / `min_window` with a `by=` projection over tumbling, sliding and session windows.
//
// The reference's `max_window(..., by)` is `reduce_window(..., partial(max, key=by))` (pysrc/bytewax/operators/
// windowing.py:2189, :2236), i.e. `fold_window(ordered=False)` (:2268-2285) with `_FoldWindowLogic` (:1692-1714) whose
// folder and merger are both `max(acc, v, key=by)`: the first on-time value seeds a window's pick, and a later value,
// in arrival order, replaces it only if by(v) > by(pick) (min: <).  Ties keep the earlier item; Python compares i64
// exactly and f64 by IEEE (NaN never wins and is never beaten, -0.0 == +0.0 is a tie), which is what one serial
// compare per value gives.  A session merge (`on_merge`, :1700-1705) is `into = max(into, orig, key=by)`: the survivor
// keeps its pick unless the merged-away session's pick is strictly better.
//
// The items themselves stay with the caller: each travels as a u64 handle with its by-value (i64 or f64 bits).  The
// per-key steps are K8's and K7's, called rather than restated: the activation is grouped by key (CUB stable sort,
// `keyed_group`) and ONE thread per key runs, item by item in arrival order, K8's late test (bw_jw_on_item, with
// bw_jw_late_rows or one LATE_SESSION_ID row for sessions) and, for an on-time item, the play: every window of
// `open_for(ts)` (bw_jw_ids / bw_jw_find_or_open), or the session `open_for` returns (bw_sess_open_for).  Then the
// session merge queue (bw_sess_merge_each) and the close (bw_jw_close_each; bw_sess_close_each + bw_sess_mids).  The
// late test never reads a window and the play never moves the clock, so one pass does both in the order the
// reference's late test, queue and unordered flush give.  `reduce_window` is always unordered: no queue, no pool.
// Notify and EOF mark the keys they wake with K8's k_jwin_mark (JwNotifyAt; AwNotifyAt for sessions) and close them.
//
// Handles are released (K8's bw_jw_release) exactly once, in the call that lets go of them: a late item's at once; a
// value that is the pick of none of its windows at once; a pick replaced in the last window holding it; the losing
// pick of a session merge; a pick when the last window holding it closes.
//
// Per key (tumbling / sliding; a key with no open window is discarded with its clock, windowing.py:1110-1113):
//   keys[slot], st[slot]   K8's table and clock state (JwTable; its JwWin array is not used)
//   win[slot * M ...]      open windows in first-opened order: id, pick's by-bits, pick's handle (24 B each)
// Per key (sessions; never discarded, windowing.py:798-806):
//   keys[slot], st[slot]   as above; kx[slot] K10's next session id and held merged ids
//   rec[slot * M ...]      sessions in id order: id, open, close, pick's by-bits and handle (40 B each)
//   mrg[slot * 2M ...]     (owner id, merged id) pairs
#pragma once
#include "../../include/bwgpu.h"
#include "bw_common.cuh"
#include "bw_jwin.cuh"
#include "bw_keyed.cuh"
#include "bw_session.cuh"
#include "bw_sjwin.cuh"

struct AwWin {  // a tumbling / sliding window
  i64 id;
  u64 by;  // the pick's by-value bits
  u64 h;   // the pick's handle
  __device__ void open(i64 i) { id = i; }  // (the caller seeds the pick)
};
struct AwSess {  // a session
  i64 id, open, close;
  u64 by, h;
};
struct AwTable {
  JwTable j;  // keys, clock state, error words, cap, M
  AwWin* win;
  AwSess* rec;
  SjKey* kx;
  i64* mrg;
  i64 gap;
  int is_max, is_f64;
  // the fail / release helpers of bw_jwin.cuh read these two
  u32* err;
  u32* why;
};
struct AwEmit {
  // closed windows: the `E` row (the pick) and its `M` row
  u64 *key, *wid, *h, *epoch, *ord, *seq, *moff, *mcnt;
  i64 *open, *close;
  u64 max_rows;
  unsigned long long* n_rows;
  i64* mids;  // merged ids of the closed sessions, [moff, moff + mcnt) per row
  unsigned long long* n_mids;
  // late items (names as JwEmit: bw_jw_late_rows)
  u64 *l_key, *l_wid, *l_epoch, *l_act, *l_row, *l_ord, *l_seq;
  u64 max_late;
  unsigned long long* n_late;
  // released handles
  u64* rel;
  u64 max_rel;
  unsigned long long* n_rel;
};

// Python's `by(v) > by(pick)` (max) / `<` (min) on i64 or f64 bits
__device__ __forceinline__ bool bw_aw_better(const AwTable& t, u64 v, u64 pick) {
  if (t.is_f64) {
    const double x = __longlong_as_double((long long)v), y = __longlong_as_double((long long)pick);
    return t.is_max ? x > y : x < y;
  }
  return t.is_max ? (i64)v > (i64)pick : (i64)v < (i64)pick;
}

// does any of the key's n windows pick h
__device__ __forceinline__ bool bw_aw_held(const AwWin* W, u32 n, u64 h) {
  for (u32 i = 0; i < n; ++i)
    if (W[i].h == h) return true;
  return false;
}

// one on-time value: `_handle_inserts` (windowing.py:1064-1077) with the fold's compare-insert in every window of
// open_for(ts), ascending id; false when the key needs more than M windows
__device__ bool bw_aw_play(const AwTable& t, const AwEmit& e, const JwParams& p, AwWin* W, u32& n, i64 ts, u64 h, u64 by) {
  i64 lo, hi;
  bw_jw_ids(p, ts, lo, hi);
  bool kept = false;
  for (i64 id = lo; id <= hi; ++id) {
    const u32 n0 = n;
    const u32 i = bw_jw_find_or_open(W, n, (u32)t.j.M, id);
    if (i == (u32)t.j.M) return false;
    AwWin& w = W[i];
    if (n > n0) {  // a new window: the value seeds its pick (shim_folder, windowing.py:2277-2281)
      w.by = by;
      w.h = h;
      kept = true;
    } else if (bw_aw_better(t, by, w.by)) {
      const u64 old = w.h;
      w.by = by;
      w.h = h;
      kept = true;
      if (!bw_aw_held(W, n, old)) bw_jw_release(t, e, old);
    }
  }
  if (!kept) bw_jw_release(t, e, h);  // the pick of none of its windows
  return true;
}

// one closed row: key, window / session id, pick, bounds, merged ids; false (and the call fails) when the emit buffer
// is full
__device__ __forceinline__ void bw_aw_emit(const AwTable& t, const AwEmit& e, const JwParams& p, u64 key, i64 id, u64 h, i64 open, i64 close,
                                           u32 cnt, const i64* MG, u32 nm, u64& seq) {
  const u64 c = atomicAdd(e.n_rows, 1ULL);
  const u64 m0 = cnt ? atomicAdd(e.n_mids, (unsigned long long)cnt) : 0;
  if (c >= e.max_rows || m0 + cnt > e.max_rows) {
    bw_jw_fail(t, BW_JW_FULL_EMIT);
    return;
  }
  e.key[c] = key;
  e.wid[c] = (u64)id;
  e.h[c] = h;
  e.open[c] = open;
  e.close[c] = close;
  e.epoch[c] = p.epoch;
  e.ord[c] = p.ord;
  e.seq[c] = seq++;
  e.moff[c] = m0;
  e.mcnt[c] = cnt;
  if (cnt) bw_sess_mids(MG, nm, id, cnt, e.mids + m0);
}

// `_handle_closed` (windowing.py:1087-1093): windows with close <= wm in first-opened order, each giving its pick; a
// pick no window still open holds is let go
__device__ void bw_aw_close(const AwTable& t, const AwEmit& e, const JwParams& p, u64 key, AwWin* W, u32& n, i64 wm) {
  u64 seq = 0;
  bw_jw_close_each(p, W, n, wm, [&](const AwWin& w) {
    const i64 cl = bw_jw_close(p, w.id);
    bw_aw_emit(t, e, p, key, w.id, w.h, cl - p.length, cl, 0, nullptr, 0, seq);
    if (!bw_aw_held(W, n, w.h)) bw_jw_release(t, e, w.h);
  });
}

// `_handle_merged` (windowing.py:1079-1085) with `on_merge` = `into = max(into, orig, key=by)`, then `close_for`
// (:774-788) at watermark wm: sessions with close < wm - gap in id order, each giving its pick and merged ids
__device__ void bw_aw_sess_finish(const AwTable& t, const AwEmit& e, const JwParams& p, u64 key, AwSess* R, i64* MG, SessWalk& w,
                                  const unsigned char* qo, const unsigned char* qt, i64 wm) {
  bw_sess_merge_each(R, w, qo, qt, [&](AwSess& into, const AwSess& orig) {
    if (bw_aw_better(t, orig.by, into.by)) {
      bw_jw_release(t, e, into.h);
      into.by = orig.by;
      into.h = orig.h;
    } else {
      bw_jw_release(t, e, orig.h);
    }
  });
  u64 seq = 0;
  bw_sess_close_each(R, MG, w.n, w.nm, bw_sess_close_after(wm, t.gap), [&](const AwSess& r, u32 cnt) {
    bw_aw_emit(t, e, p, key, r.id, r.h, r.open, r.close, cnt, MG, w.nm, seq);
    bw_jw_release(t, e, r.h);
  });
}

// one thread per key segment, tumbling / sliding: per item in arrival order K8's late test, then the play of an
// on-time item; then the close at the watermark after the key's last item
__global__ void k_awin_apply(AwTable t, AwEmit e, JwParams p, const u64* ksorted, const u32* isorted, const u32* headpos, const u64* handles,
                             const u64* by, const i64* ts_us, u64 n) {
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.j.keys, t.j.cap, key, t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      continue;
    }
    JwState st = t.j.st[s];
    bw_jw_begin(st, p);
    AwWin* W = t.win + s * (u64)t.j.M;
    u32 nw = st.n;
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0;
    bool full = false;
    for (u64 q = h; q < n && ksorted[q] == key && !full; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      if (bw_jw_on_item(st, p, ts, wm)) {  // late: one row per id of late_for(ts); the handle is let go
        bw_jw_late_rows(t, e, p, key, ts, o, lseq);
        bw_jw_release(t, e, handles[o]);
      } else {
        full = !bw_aw_play(t, e, p, W, nw, ts, handles[o], by[o]);
      }
    }
    if (full) {
      bw_jw_fail(t, BW_JW_FULL_WINDOWS);
      continue;  // the call fails and the step refuses further work
    }
    st.wm = wm;
    st.act = p.ord;
    bw_aw_close(t, e, p, key, W, nw, wm);
    st.n = nw;
    if (nw == 0) st.init = 0;  // _is_empty (windowing.py:1110-1113): the engine discards the logic, clock included
    t.j.st[s] = st;
  }
}

// one thread per key segment, sessions: per item K8's late test (one row, window LATE_SESSION_ID, windowing.py:764-766)
// or open_for and the compare-insert into the session it returns, even one a merge just took away (:1064-1077); then
// the merge queue and the close
__global__ void k_aswin_apply(AwTable t, AwEmit e, JwParams p, const u64* ksorted, const u32* isorted, const u32* headpos, const u64* handles,
                              const u64* by, const i64* ts_us, u64 n) {
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.j.keys, t.j.cap, key, t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      continue;
    }
    JwState st = t.j.st[s];
    bw_jw_begin(st, p);  // (kx starts at zero: k_awin_init)
    AwSess* R = t.rec + s * (u64)t.j.M;
    i64* MG = t.mrg + s * (u64)(2 * t.j.M);
    SjKey kx = t.kx[s];
    unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
    SessWalk w;
    bw_sess_walk_begin(w, st.n, kx.nm);
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0;
    bool full = false;
    for (u64 q = h; q < n && ksorted[q] == key; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      const u64 hv = handles[o];
      if (bw_jw_on_item(st, p, ts, wm)) {
        const u64 i = atomicAdd(e.n_late, 1ULL);
        if (i >= e.max_late) {
          bw_jw_fail(t, BW_JW_FULL_LATE);
        } else {
          e.l_key[i] = key;
          e.l_wid[i] = (u64)BW_SESS_LATE_ID;
          e.l_epoch[i] = p.epoch;
          e.l_act[i] = p.batch_no;
          e.l_row[i] = o;
          e.l_ord[i] = p.ord;
          e.l_seq[i] = lseq++;
        }
        bw_jw_release(t, e, hv);
        continue;
      }
      bool fresh;
      const int i = bw_sess_open_for(R, MG, w, qo, qt, t.j.M, t.gap, ts, fresh);
      if (i < 0) {
        full = true;
        break;
      }
      AwSess& r = R[i];
      const u64 b = by[o];
      if (fresh) {  // a new session, id max_key + 1, seeded with the value
        r.id = kx.next_id++;
        r.open = r.close = ts;
        r.by = b;
        r.h = hv;
      } else if (bw_aw_better(t, b, r.by)) {
        bw_jw_release(t, e, r.h);
        r.by = b;
        r.h = hv;
      } else {
        bw_jw_release(t, e, hv);
      }
    }
    if (full) {
      bw_jw_fail(t, BW_JW_FULL_WINDOWS);
      continue;
    }
    st.wm = wm;
    st.act = p.ord;
    bw_aw_sess_finish(t, e, p, key, R, MG, w, qo, qt, wm);
    st.n = w.n;
    kx.nm = w.nm;
    t.kx[s] = kx;
    t.j.st[s] = st;
  }
}

// notify_at of the session windower (windowing.py:790-796, :1153-1180 with an identity `to_system_utc`): the earliest
// close + gap
struct AwNotifyAt {
  i64 gap;
  __device__ __forceinline__ i64 operator()(const JwParams&, const JwState& st, const AwSess* R) const {
    i64 at = INT64_MAX;
    for (u32 i = 0; i < st.n; ++i) {
      const i64 c = R[i].close + gap;  // close <= UTC_MAX and gap <= UTC_MAX - UTC_MIN: no overflow
      at = c < at ? c : at;
    }
    return at;
  }
};

// notify / EOF, one thread per slot: a key k_jwin_mark woke closes what its watermark allows
__global__ void k_awin_close(AwTable t, AwEmit e, JwParams p, int session) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.j.cap; s += (u64)gridDim.x * blockDim.x) {
    JwState st = t.j.st[s];
    if (!st.init || st.act != p.ord) continue;
    const u64 key = t.j.keys[s];
    if (session) {
      AwSess* R = t.rec + s * (u64)t.j.M;
      i64* MG = t.mrg + s * (u64)(2 * t.j.M);
      SjKey kx = t.kx[s];
      u64 seq = 0;
      bw_sess_close_each(R, MG, st.n, kx.nm, bw_sess_close_after(st.wm, t.gap), [&](const AwSess& r, u32 cnt) {
        bw_aw_emit(t, e, p, key, r.id, r.h, r.open, r.close, cnt, MG, kx.nm, seq);
        bw_jw_release(t, e, r.h);
      });
      t.kx[s] = kx;
    } else {
      u32 nw = st.n;
      bw_aw_close(t, e, p, key, t.win + s * (u64)t.j.M, nw, st.wm);
      st.n = nw;
      if (nw == 0) st.init = 0;  // discarded with its clock (windowing.py:1110-1113)
    }
    t.j.st[s] = st;
  }
}

__global__ void k_awin_init(AwTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.j.cap; s += (u64)gridDim.x * blockDim.x) {
    t.j.keys[s] = BW_EMPTY_KEY;
    t.j.st[s].init = 0;
    t.j.st[s].n = t.j.st[s].nq = 0;
    t.j.st[s].qord = ~0ULL;
    t.j.st[s].act = ~0ULL;
    if (t.kx) {
      t.kx[s].next_id = 0;
      t.kx[s].nm = 0;
    }
  }
}
