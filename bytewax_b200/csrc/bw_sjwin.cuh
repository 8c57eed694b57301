// bw_sjwin.cuh -- K10: `join_window` with insert modes first / last over `SessionWindower`.
//
// The reference runs `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) over
// `_SessionWindowerLogic` (:671-810) with one `_JoinWindowLogic` (:1849-1902) per session: per key, in arrival order,
// the EventClock's late test; the queue; `_flush_queue` (:1095-1108); `open_for` per due value and the join step on the
// session it returned; the merge queue (`on_merge`, :1879-1891); `close_for` in id order.  This is K7's session walk
// (bw_session.cuh: open_for, _session_find_merges, the merge queue, close_for -- called, not copied) with K8's join
// state and queue machinery (bw_jwin.cuh: clock, late test, pool, pool sort, carry-over, notify marking, release).
//
// Unordered mode: k_sjwin_apply, one thread per key, runs the late test, plays the on-time items in arrival order,
// then the merges and the close.  Ordered mode: k_sjwin_apply runs the late test and appends on-time items to K8's
// pool; K8's two stable radix passes put the due entries in play order; k_sjwin_flush, one thread per slot, plays
// them, carries the rest over (bw_jw_carry), merges and closes.  Notify and EOF mark the keys they wake (K8's
// k_jwin_mark with SjNotifyAt) and run the same flush.
//
// Merges (`on_merge(into = survivor, orig)`): "first" does `into.state |= orig.state` (where orig's side is set, it
// wins), "last" `orig.state |= into.state; into.state = orig.state` (where the survivor's side is set, it wins); then
// "complete" emits under the survivor's id and clears once every side is set, "running" emits.
//
// A handle sits in at most one side of one session, so it is released (K8's bw_jw_release) exactly once: a late item's
// in the call that received it; a "first" value that found its side set at once; a value replaced by "last"; every
// handle of a state "complete" emits and clears; the losing handle of a side both merged sessions set; and every
// handle of a session when it closes.
//
// Per key, never freed (session state is never discarded, windowing.py:798-806, so the clock survives the sessions):
//   keys[slot]                 the key (bw_keyed_find table; slot `cap` is the BW_EMPTY_KEY alias slot)
//   st[slot]                   K8's JwState: the EventClock pair, the flush watermark and call, live sessions n, queue
//   kx[slot]                   next session id, held merged ids
//   rec[slot * M ...]          sessions (id, set mask, 4 handles, open, close) in id order == the reference's dict order
//   mrg[slot * 2M ...]         (owner id, merged id) pairs, the `merged_ids` sets of the live sessions
#pragma once
#include "../../include/bwgpu.h"
#include "bw_common.cuh"
#include "bw_jwin.cuh"
#include "bw_keyed.cuh"
#include "bw_session.cuh"

// a session: K8's join state (id, mask, handles: so bw_jw_emit ships it as is) and the session's bounds.  (`open` the
// bound hides JwWin::open, which only K8's window lookup calls.)
struct __align__(16) SjRec : JwWin {
  i64 open, close;
};
struct SjKey {
  i64 next_id;  // max_key + 1 (never resets)
  u32 nm, pad;  // held merged ids
};
struct SjTable : JwTable {  // K8's keys, clock / queue state, error words, cap, M (= max_sessions_per_key), sides
  SjRec* rec;
  SjKey* kx;
  i64* mrg;
  i64 gap;
};
struct SjEmit : JwEmit {  // K8's down, late, release and carry-over buffers (late window id: LATE_SESSION_ID)
  // meta rows: WindowMetadata(open, close, merged_ids)
  i64 *m_open, *m_close;
  u64 *m_moff, *m_mcnt;
  i64* mids;  // merged ids of the meta rows, [moff, moff + mcnt) per row
  unsigned long long* n_mids;
};

// notify_at (windowing.py:1153-1180 with an identity `to_system_utc`; the windower's :790-796): the earliest close +
// gap, or, ordered, the ts of queue[0] if that is sooner (R: SjRec here, ScRec in bw_scwin.cuh)
struct SjNotifyAt {
  i64 gap;
  template <class R>
  __device__ __forceinline__ i64 operator()(const JwParams& p, const JwState& st, const R* Rs) const {
    i64 at = INT64_MAX;
    for (u32 i = 0; i < st.n; ++i) {
      const i64 c = Rs[i].close + gap;  // close <= UTC_MAX and gap <= UTC_MAX - UTC_MIN: no overflow
      at = c < at ? c : at;
    }
    if (p.ordered && st.nq && st.q0ts < at) at = st.q0ts;
    return at;
  }
};

// `_check_emit` after a value or a merge: "complete" emits and clears (`_JoinState.clear`) once every side is set,
// "running" emits always
__device__ void bw_sj_check_emit(const SjTable& t, const SjEmit& e, const JwParams& p, u64 key, SjRec& r, u64& seq) {
  if (p.emit_mode == BW_JOIN_EMIT_COMPLETE) {
    if (r.mask == (1ULL << t.sides) - 1) {
      bw_jw_emit(t, e, p, key, r, seq);
      for (int s = 0; s < t.sides; ++s) bw_jw_release(t, e, r.h[s]);
      r.mask = 0;
    }
  } else if (p.emit_mode == BW_JOIN_EMIT_RUNNING) {
    bw_jw_emit(t, e, p, key, r, seq);
  }
}

// one due value: open_for (K7's walk), then `_JoinWindowLogic.on_value` (windowing.py:1866-1876) on the session it
// returned; false when the key needs more than M sessions or merged ids
__device__ bool bw_sj_play(const SjTable& t, const SjEmit& e, const JwParams& p, u64 key, SjRec* R, i64* MG, SessWalk& w, unsigned char* qo,
                           unsigned char* qt, SjKey& kx, i64 ts, u64 h, int side, u64& seq) {
  bool fresh;
  const int i = bw_sess_open_for(R, MG, w, qo, qt, t.M, t.gap, ts, fresh);
  if (i < 0) return false;
  SjRec& r = R[i];
  if (fresh) {  // a new session, id max_key + 1, with builder(None): an empty join state
    r.id = kx.next_id++;
    r.open = r.close = ts;
    r.mask = 0;
  }
  const u64 bit = 1ULL << side;
  if (!(r.mask & bit)) {
    r.h[side] = h;
    r.mask |= bit;
  } else if (p.insert_last) {
    bw_jw_release(t, e, r.h[side]);
    r.h[side] = h;
  } else {
    bw_jw_release(t, e, h);  // "first": the side stays as it was
  }
  bw_sj_check_emit(t, e, p, key, r, seq);
  return true;
}

// `_handle_merged` (windowing.py:1079-1085) with `on_merge` (:1879-1891), then `_handle_closed` (:1087-1093) at
// watermark wm: `final` row, then the meta row, of each closing session in id order
__device__ void bw_sj_finish(const SjTable& t, const SjEmit& e, const JwParams& p, u64 key, SjRec* R, i64* MG, SessWalk& w,
                             const unsigned char* qo, const unsigned char* qt, i64 wm, u64& seq) {
  bw_sess_merge_each(R, w, qo, qt, [&](SjRec& into, const SjRec& orig) {
    for (int s = 0; s < t.sides; ++s) {
      if (!(orig.mask >> s & 1)) continue;
      if (!(into.mask >> s & 1)) {
        into.h[s] = orig.h[s];
        into.mask |= 1ULL << s;
      } else if (p.insert_last) {
        bw_jw_release(t, e, orig.h[s]);  // the survivor's value wins
      } else {
        bw_jw_release(t, e, into.h[s]);  // the merged-away session's value wins
        into.h[s] = orig.h[s];
      }
    }
    bw_sj_check_emit(t, e, p, key, into, seq);
  });
  u64 mseq = 0;
  bw_sess_close_each(R, MG, w.n, w.nm, bw_sess_close_after(wm, t.gap), [&](const SjRec& r, u32 cnt) {
    if (p.emit_mode == BW_JOIN_EMIT_FINAL) bw_jw_emit(t, e, p, key, r, seq);
    const u64 m = atomicAdd(e.n_meta, 1ULL);
    const u64 m0 = cnt ? atomicAdd(e.n_mids, (unsigned long long)cnt) : 0;
    if (m >= e.max_rows || m0 + cnt > e.max_rows) {
      bw_jw_fail(t, BW_JW_FULL_EMIT);
    } else {
      e.m_key[m] = key;
      e.m_wid[m] = (u64)r.id;
      e.m_open[m] = r.open;
      e.m_close[m] = r.close;
      e.m_epoch[m] = p.epoch;
      e.m_ord[m] = p.ord;
      e.m_seq[m] = mseq++;
      e.m_moff[m] = m0;
      e.m_mcnt[m] = cnt;
      bw_sess_mids(MG, w.nm, r.id, cnt, e.mids + m0);
    }
    for (int s = 0; s < t.sides; ++s)
      if (r.mask >> s & 1) bw_jw_release(t, e, r.h[s]);
  });
}

// pass A, one thread per key segment: the late test per item (windowing.py:1115-1133, :263-287; a late item gives one
// row, window LATE_SESSION_ID, :764-766).  Unordered: then the play of the on-time items in arrival order, the merges
// and the close.  Ordered: the on-time items go to K8's pool at base + q.
__global__ void k_sjwin_apply(SjTable t, SjEmit e, JwParams p, JwPool pool, u64 base, const u64* ksorted, const u32* isorted,
                              const u32* headpos, const u64* handles, const unsigned char* sides, const i64* ts_us, unsigned char* late,
                              u64 n) {
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.keys, t.cap, key, t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      // the call fails; the pool sort and flush that follow read this key's entries as late items' (as K8 does)
      for (u64 q = h; q < n && ksorted[q] == key; ++q)
        if (p.ordered) {
          pool.slot[base + q] = (u32)t.cap;
          pool.side[base + q] = (unsigned char)BW_JW_DROP;
        }
      continue;
    }
    JwState st = t.st[s];
    bw_jw_begin(st, p);  // (kx starts at zero: k_sjwin_init)
    u64 end = h;
    while (end < n && ksorted[end] == key) ++end;
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0;
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
      if (is_late) {  // the late row; the handle is let go
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
      SjRec* R = t.rec + s * (u64)t.M;
      i64* MG = t.mrg + s * (u64)(2 * t.M);
      SjKey kx = t.kx[s];
      unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
      SessWalk w;
      bw_sess_walk_begin(w, st.n, kx.nm);
      u64 seq = 0;
      bool full = false;
      for (u64 q = h; q < end && !full; ++q) {
        if (late[q]) continue;
        const u32 o = isorted[q];
        full = !bw_sj_play(t, e, p, key, R, MG, w, qo, qt, kx, ts_us[o], handles[o], sides[o], seq);
      }
      if (full) {
        bw_jw_fail(t, BW_JW_FULL_WINDOWS);
        continue;  // the call fails and the join refuses further work: no row of this key is emitted half-done
      }
      bw_sj_finish(t, e, p, key, R, MG, w, qo, qt, wm, seq);
      st.n = w.n;
      kx.nm = w.nm;
      t.kx[s] = kx;
    }
    t.st[s] = st;
  }
}

// pass B, one thread per slot: a woken key plays its due entries (in ts order, ties in arrival order), keeps the
// others queued in arrival order, merges and closes; an idle key's entries move to the next pool unchanged.  Also the
// notify / EOF flush of unordered mode (perm NULL: nothing queued).
__global__ void k_sjwin_flush(SjTable t, SjEmit e, JwParams p, JwPool pool, const u32* perm) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    JwState st = t.st[s];
    if (!st.init) continue;
    const bool woken = st.act == p.ord;
    const u32 qb = st.qord == p.ord ? st.qb : 0, qe = st.qord == p.ord ? st.qe : 0;
    if (!woken && qb == qe) continue;
    const u64 key = t.keys[s];
    SjRec* R = t.rec + s * (u64)t.M;
    i64* MG = t.mrg + s * (u64)(2 * t.M);
    SjKey kx = t.kx[s];
    unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
    SessWalk w;
    bw_sess_walk_begin(w, st.n, kx.nm);
    u64 seq = 0;
    u32 keep = 0;
    bool full = false;
    for (u32 i = qb; i < qe; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] == BW_JW_DROP) continue;
      if (woken && pool.ts[x] <= st.wm) {
        if (!full) full = !bw_sj_play(t, e, p, key, R, MG, w, qo, qt, kx, pool.ts[x], pool.h[x], pool.side[x], seq);
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
      bw_sj_finish(t, e, p, key, R, MG, w, qo, qt, st.wm, seq);
      st.n = w.n;
      kx.nm = w.nm;
      t.kx[s] = kx;
    }
    t.st[s] = st;
  }
}

__global__ void k_sjwin_init(SjTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.keys[s] = BW_EMPTY_KEY;
    t.st[s].init = 0;
    t.st[s].n = t.st[s].nq = 0;
    t.st[s].qord = ~0ULL;
    t.st[s].act = ~0ULL;
    t.kx[s].next_id = 0;
    t.kx[s].nm = 0;
  }
}
