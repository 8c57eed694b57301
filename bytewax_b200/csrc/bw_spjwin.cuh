// bw_spjwin.cuh -- K16: `join_window` with insert mode product over `SessionWindower`.
//
// The reference runs `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) over
// `_SessionWindowerLogic` (:671-810) with one `_JoinWindowLogic` (:1849-1902) per session whose `_JoinState`
// (operators/__init__.py:2072-2120) keeps one list per side.  Per key, per call: `_handle_inserts` -- `open_for` and
// `add_val` per due value, "complete" emitting the product and clearing once every side is non-empty, "running" after
// every value; `_handle_merged` -- per queued merge, in discovery order, `into.state += orig.state` (per side the
// survivor's list, then the merged-away session's), then "complete" / "running" as after a value, under the survivor's
// id; `_handle_closed` -- the `final` product and the meta row of each closing session, in id order.
//
// The per-key steps are called, not restated: K8's clock, late test, pool, pool sort, carry-over and notify marking
// (bw_jwin.cuh), K10's session walk (bw_session.cuh: open_for, _session_find_merges, the merge queue, close_for with
// merged ids) and its notify_at (SjNotifyAt), K14's emission events, stage records, ordering and expansion
// (bw_pjwin.cuh), K9's entry store and its compaction.  Unordered: k_spjwin_apply, one thread per key, runs the late test,
// plays the on-time values in arrival order, merges and closes.  Ordered: k_spjwin_apply runs the late test and fills
// K8's pool; K8's sort puts the due entries in play order; k_spjwin_flush, one thread per slot, plays them, carries the
// rest over, merges and closes.  Notify and EOF mark the keys with K8's k_jwin_mark and run the same flush.
//
// A session's lists are K14's: one entry per played value in K9's ENTRY STORE -- its session's cell and side in the
// reference word, its rank within (cell, side), the handle -- and per cell and side a count and the first rank of the
// current generation, so each list is the ranks [gen, cnt).  An emission appends K14's EVENT (a rank range per side),
// and every cell that emits in a call gets one STAGE RECORD, the union of its events' ranges.
//
// A merge of B into A copies nothing: per side, B's live ranks [genB, cntB) become A's ranks [cntA, cntA + cntB - genB),
// A's count grows by cntB - genB, and B's cell records ONE HOP -- the cell it went to, the call, genB and cntA (where
// its list starts in A's).  Only one hop, because a value may have to be staged under several coordinates in one call:
// under a chain B -> A -> X a value of B is emitted as B's rank, then as A's at (B -> A), then as X's at (A -> X).
//
// k_spjwin_gather, over the whole store, after the per-key kernels of every call that emitted, merged or closed: per
// entry, starting at its (cell, rank), (1) a stage record of this call on the cell that covers the rank gets the handle;
// (2) a cell merged away in this call ends the entry when the rank is below that hop's gen (a "complete" clear before the
// merge), else the rank moves to the hop's cell, rank - gen + base, and the walk repeats (at most M hops); (3) at the last
// cell the entry dies when its session closed in this call or its rank is below the cell's gen, and is retagged there
// otherwise.  A dead entry releases its handle: a value sits in one session, so it has exactly one entry.  A cell merged
// away in a call is free again only after that call's gather: the walk never reuses a cell of a record it holds.
//
// Handles: a value's is released in the call its entry dies in (cleared, closed), a late item's in the call that received
// it.  Session state is never discarded (:798-806), so the clock outlives the sessions.
//
// Per key (slot), never freed:
//   keys[slot], st[slot]     as K8 (JwTable; its JwWin array is not used)
//   kx[slot]                 next session id, held merged ids
//   rec[slot * M ...]        sessions (id, open, close, cell) in id order == the reference's dict order
//   mrg[slot * 2M ...]       (owner id, merged id) pairs, the `merged_ids` sets of the live sessions (K10)
// Per cell (slot * M + cell): K14's counts and generations, stage record (rec_ord / rec_c) and close call (close_ord);
//   mord / hop: the call in which the session on the cell was merged away, and that merge's hop.
#pragma once
#include "../../include/bwgpu.h"
#include "bw_collect.cuh"
#include "bw_pjwin.cuh"
#include "bw_session.cuh"
#include "bw_sjwin.cuh"

struct __align__(16) SpRec {
  i64 id, open, close;
  u32 cell, pad;
};
struct SpKey {
  i64 next_id;  // max_key + 1 (never resets)
  u32 nm, pad;  // held merged ids
};
struct SpHop {  // a merge of the session on this cell into the one on `into`
  u64 into;
  u32 gen[BW_JW_MAXSIDES];   // the merged-away lists started at these ranks ...
  u32 base[BW_JW_MAXSIDES];  // ... and go on at these ranks of `into`'s lists
};
struct SpTable : PjTable {  // K14's keys, clock / queue state, cells, stage records, close calls, error words
  SpRec* rec;
  SpKey* kx;
  i64* mrg;
  u64* mord;
  SpHop* hop;
  i64 gap;
};
struct SpEmit : PjEmit {  // K14's events, meta rows, late rows (window id LATE_SESSION_ID), releases, carry-over, staging
  // meta rows: WindowMetadata(open, close, merged_ids)
  i64 *m_open, *m_close;
  u64 *m_moff, *m_mcnt;
  i64* mids;  // merged ids of the meta rows, [moff, moff + mcnt) per row
  unsigned long long* n_mids;
  unsigned long long* n_mrg;  // merges applied so far (the gather runs after a call that merged)
};

// reserve `n` store entries for one key; false (and the call fails) when they do not fit
__device__ __forceinline__ bool bw_sp_reserve(const SpTable& t, const CwStore& es, u64 n, u64& at) {
  at = n ? atomicAdd(es.n, (unsigned long long)n) : 0;
  if (at + n <= es.cap) return true;
  bw_jw_fail(t, BW_CW_FULL_STORE);  // (sized by the host for every value a call can play: never reached)
  return false;
}

// `_check_emit` after a value or a merge: "complete" emits the product and clears once every side is non-empty,
// "running" emits always (K14's event and stage record, under the session's id)
__device__ void bw_sp_check_emit(const SpTable& t, const SpEmit& e, const JwParams& p, u64 key, u64 slot, const SpRec& r, u64& seq,
                                 u64& touched) {
  const PjWin w{r.id, r.cell, 0};
  if (p.emit_mode == BW_JOIN_EMIT_COMPLETE) {
    PjCell& c = t.cell[slot * (u64)t.j.M + r.cell];
    bool all = true;
    for (int s = 0; s < t.j.sides; ++s) all = all && c.cnt[s] > c.gen[s];
    if (all) {
      bw_pj_emit(t, e, p, key, slot, w, seq, touched);
      for (int s = 0; s < t.j.sides; ++s) c.gen[s] = c.cnt[s];  // _JoinState.clear
    }
  } else if (p.emit_mode == BW_JOIN_EMIT_RUNNING) {
    bw_pj_emit(t, e, p, key, slot, w, seq, touched);
  }
}

// one due value: open_for (K10's walk), then `add_val` and `on_value` on the session it returned, even one its own
// find_merges just took away (windowing.py:1064-1077): the value's entry goes to es[ei++]; 0, or the BW_* reason the key
// cannot go on
__device__ u32 bw_sp_play(const SpTable& t, const SpEmit& e, const CwStore& es, const JwParams& p, u64 key, u64 slot, SpRec* R, i64* MG,
                          SessWalk& w, unsigned char* qo, unsigned char* qt, SpKey& kx, i64 ts, u64 h, int side, u64& ei, u64& seq,
                          u64& touched) {
  const u32 M = (u32)t.j.M;
  bool fresh;
  const int i = bw_sess_open_for(R, MG, w, qo, qt, (int)M, t.gap, ts, fresh);
  if (i < 0) return BW_JW_FULL_WINDOWS;
  SpRec& r = R[i];
  const u64 c0 = slot * M;
  if (fresh) {  // a new session, id max_key + 1, on the lowest cell no record the key holds has, with empty lists
    u64 used = 0;
    for (u32 k = 0; k + 1 < w.n; ++k) used |= 1ULL << R[k].cell;
    r.id = kx.next_id++;
    r.open = r.close = ts;
    r.cell = (u32)__ffsll((long long)~used) - 1;
    t.cell[c0 + r.cell] = PjCell{};
  }
  PjCell& c = t.cell[c0 + r.cell];
  if (c.cnt[side] == 0xFFFFFFFFu) return BW_PJ_FULL_SIDE;
  es.ref[ei] = ((c0 + r.cell) << 2) | (u64)side;
  es.rank[ei] = c.cnt[side]++;
  es.h[ei] = h;
  ++ei;
  bw_sp_check_emit(t, e, p, key, slot, r, seq, touched);
  return 0;
}

// `_handle_merged` (windowing.py:1079-1085) with `on_merge` (:1879-1891), then `_handle_closed` (:1087-1093) at
// watermark wm: the `final` event, then the meta row, of each closing session in id order; then the stage records'
// staging ranges.  0, or the BW_* reason the key cannot go on.
__device__ u32 bw_sp_finish(const SpTable& t, const SpEmit& e, const JwParams& p, u64 key, u64 slot, SpRec* R, i64* MG, SessWalk& w,
                            const unsigned char* qo, const unsigned char* qt, SpKey& kx, i64 wm, u64& seq, u64& touched) {
  const u64 c0 = slot * (u64)t.j.M;
  const int sides = t.j.sides;
  u32 bad = 0;
  const bool merges = w.nq != 0;
  bw_sess_merge_each(R, w, qo, qt, [&](SpRec& into, const SpRec& orig) {
    const u64 ic = c0 + into.cell, oc = c0 + orig.cell;
    PjCell& a = t.cell[ic];
    const PjCell b = t.cell[oc];
    SpHop x;
    x.into = ic;
    for (int s = 0; s < BW_JW_MAXSIDES; ++s) {
      x.gen[s] = b.gen[s];
      x.base[s] = a.cnt[s];
      if (s >= sides) continue;
      const u32 moved = b.cnt[s] - b.gen[s];
      if (moved > 0xFFFFFFFFu - a.cnt[s]) bad = BW_PJ_FULL_SIDE;
      else a.cnt[s] += moved;
    }
    t.hop[oc] = x;
    t.mord[oc] = p.ord;
    bw_sp_check_emit(t, e, p, key, slot, into, seq, touched);
  });
  if (bad) return bad;
  if (merges) atomicAdd(e.n_mrg, 1ULL);
  u64 mseq = 0;
  bw_sess_close_each(R, MG, w.n, w.nm, bw_sess_close_after(wm, t.gap), [&](const SpRec& r, u32 cnt) {
    if (p.emit_mode == BW_JOIN_EMIT_FINAL) bw_pj_emit(t, e, p, key, slot, PjWin{r.id, r.cell, 0}, seq, touched);
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
    t.close_ord[c0 + r.cell] = p.ord;  // its entries die in this call's gather
  });
  kx.nm = w.nm;
  bw_pj_stage(t, e, slot, touched);
  return 0;
}

// pass A, one thread per key segment: K8's late test per item; unordered, then the play of the on-time items in arrival
// order, the merges and the close; ordered, the on-time items go to K8's pool at base + q
__global__ void k_spjwin_apply(SpTable t, SpEmit e, CwStore es, JwParams p, JwPool pool, u64 base, const u64* ksorted, const u32* isorted,
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
    bw_jw_begin(st, p);  // (kx starts at zero: k_spjwin_init)
    u64 end = h;
    while (end < n && ksorted[end] == key) ++end;
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0, entries = 0;
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
      if (is_late) {  // one row, window LATE_SESSION_ID (windowing.py:764-766, :1125-1127); the handle is let go
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
      } else {
        ++entries;
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
      u64 ei;
      if (!bw_sp_reserve(t, es, entries, ei)) continue;
      const u64 eend = ei + entries;
      SpRec* R = t.rec + s * (u64)t.j.M;
      i64* MG = t.mrg + s * (u64)(2 * t.j.M);
      SpKey kx = t.kx[s];
      unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
      SessWalk w;
      bw_sess_walk_begin(w, st.n, kx.nm);
      u64 seq = 0, touched = 0;
      u32 bad = 0;
      for (u64 q = h; q < end && !bad; ++q) {
        if (late[q]) continue;
        const u32 o = isorted[q];
        bad = bw_sp_play(t, e, es, p, key, s, R, MG, w, qo, qt, kx, ts_us[o], handles[o], sides[o], ei, seq, touched);
      }
      if (!bad) bad = bw_sp_finish(t, e, p, key, s, R, MG, w, qo, qt, kx, wm, seq, touched);
      if (bad) {
        bw_cw_kill(es, ei, eend);
        bw_jw_fail(t, bad);
        continue;  // the call fails and the join refuses further work: no row of this key is emitted half-done
      }
      st.n = w.n;
      t.kx[s] = kx;
    }
    t.j.st[s] = st;
  }
}

// pass B, one thread per slot: a woken key plays its due entries (in ts order, ties in arrival order), keeps the others
// queued in arrival order, merges and closes; an idle key's entries move to the next pool unchanged.  Also the notify /
// EOF flush of unordered mode (nothing queued).
__global__ void k_spjwin_flush(SpTable t, SpEmit e, CwStore es, JwParams p, JwPool pool, const u32* perm) {
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
      if (woken && pool.ts[x] <= st.wm) ++entries;
      else ++keep;
    }
    u64 ei;
    if (!bw_sp_reserve(t, es, entries, ei)) continue;
    const u64 eend = ei + entries;
    const u64 key = t.j.keys[s];
    SpRec* R = t.rec + s * (u64)t.j.M;
    i64* MG = t.mrg + s * (u64)(2 * t.j.M);
    SpKey kx = t.kx[s];
    unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
    SessWalk w;
    bw_sess_walk_begin(w, st.n, kx.nm);
    u64 seq = 0, touched = 0;
    u32 bad = 0;
    for (u32 i = qb; i < qe && !bad; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] != BW_JW_DROP && woken && pool.ts[x] <= st.wm)
        bad = bw_sp_play(t, e, es, p, key, s, R, MG, w, qo, qt, kx, pool.ts[x], pool.h[x], pool.side[x], ei, seq, touched);
    }
    if (!bad && woken) bad = bw_sp_finish(t, e, p, key, s, R, MG, w, qo, qt, kx, st.wm, seq, touched);
    if (bad) {
      bw_cw_kill(es, ei, eend);
      bw_jw_fail(t, bad);
      continue;
    }
    if (keep && !bw_jw_carry(t, e, pool, perm, qb, qe, woken, s, keep, st)) continue;
    st.nq = keep;
    if (woken) {
      st.n = w.n;
      t.kx[s] = kx;
    }
    t.j.st[s] = st;
  }
}

// after the per-key kernels of a call that emitted, merged or closed (rec0 / meta0 / mrg0: the counts before it), over
// the whole store: each entry is staged by every stage record of this call along its hops, then dies (releasing its
// handle) or is retagged to the cell its values went to.  Nothing to do after a failed call (records may lack staging).
__global__ void k_spjwin_gather(SpTable t, SpEmit e, CwStore es, JwParams p, u64 rec0, u64 meta0, u64 mrg0, unsigned long long* n_dead) {
  if (*t.err) return;
  if (*e.n_rec == rec0 && *e.n_meta == meta0 && *e.n_mrg == mrg0) return;
  const u64 n = *es.n;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  for (u64 b = (u64)blockIdx.x * blockDim.x; b < n; b += stride) {  // (b is warp-uniform: the whole warp reaches the ballot)
    const u64 i = b + threadIdx.x;
    bool dead = false;
    u64 h = 0;
    if (i < n) {
      const u64 r = es.ref[i];
      if (r != BW_CW_DEAD) {
        u64 cell = r >> 2;
        const int s = (int)(r & 3);
        u32 rank = es.rank[i];
        h = es.h[i];
        bool moved = false;
        for (int hop = 0; hop <= BW_SESS_MAXM; ++hop) {  // (a chain within one call has fewer than M hops)
          if (t.rec_ord[cell] == p.ord) {
            const u64 c = t.rec_c[cell];
            const u32 d = rank - e.rb[c * 4 + s];  // (wraps above every count when rank < b)
            if (d < e.rn[c * 4 + s]) e.stage[e.rbase[c * 4 + s] + d] = h;
          }
          if (t.mord[cell] != p.ord) break;
          const SpHop& x = t.hop[cell];
          if (rank < x.gen[s]) {  // cleared before the merge: not in the list that moved
            dead = true;
            break;
          }
          rank = rank - x.gen[s] + x.base[s];
          cell = x.into;
          moved = true;
        }
        if (!dead) dead = t.close_ord[cell] == p.ord || rank < t.cell[cell].gen[s];
        if (dead) {
          es.ref[i] = BW_CW_DEAD;
        } else if (moved) {
          es.ref[i] = (cell << 2) | (u64)s;
          es.rank[i] = rank;
        }
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, dead);
    if (!m) continue;
    u64 at = 0;
    if (lane == (unsigned)__ffs(m) - 1) {
      at = atomicAdd(e.n_rel, (unsigned long long)__popc(m));
      atomicAdd(n_dead, (unsigned long long)__popc(m));
    }
    at = __shfl_sync(0xffffffffu, at, __ffs(m) - 1) + __popc(m & ((1u << lane) - 1));
    if (dead) {
      if (at < e.max_rel) e.rel[at] = h;  // (sized by the host for every handle the call can release: never reached)
      else bw_jw_fail(t, BW_JW_FULL_EMIT);
    }
  }
}

__global__ void k_spjwin_init(SpTable t) {
  const u64 cells = (t.j.cap + 1) * (u64)t.j.M;
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < cells; s += (u64)gridDim.x * blockDim.x) {
    t.rec_ord[s] = ~0ULL;
    t.close_ord[s] = ~0ULL;
    t.mord[s] = ~0ULL;
    if (s > t.j.cap) continue;
    t.j.keys[s] = BW_EMPTY_KEY;
    t.j.st[s].init = 0;
    t.j.st[s].n = t.j.st[s].nq = 0;
    t.j.st[s].qord = ~0ULL;
    t.j.st[s].act = ~0ULL;
    t.kx[s].next_id = 0;
    t.kx[s].nm = 0;
  }
}
