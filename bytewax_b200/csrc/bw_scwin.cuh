// bw_scwin.cuh -- K12: `collect_window` into list / set / dict over `SessionWindower`.
//
// The reference runs `_WindowLogic.on_batch` (pysrc/bytewax/operators/windowing.py:1115-1133) over
// `_SessionWindowerLogic` (:671-810) with one `_FoldWindowLogic` (:1692-1714) per session whose folder appends, adds or
// sets each value and whose merger is `list.__add__` / `set.union` / `_collect_dict_merger` (`_collect_get_callbacks`,
// :1356-1384), called as `into.state = merger(into.state, gone.state)`.  A session's state is therefore its values in
// play order with every merged-away session's values spliced in, as a block, where the merge happened.  The device
// keeps the values as handles in K9's ENTRY STORE (bw_collect.cuh) and the merge structure as INTERVALS; the host builds
// each container from its handles and applies the merger at each interval, so sets iterate as the reference's do.
//
// The per-key steps are called, not restated: K8's clock, late test, pool, pool sort, carry-over and notify marking
// (bw_jwin.cuh), K10's session walk (bw_session.cuh: open_for, _session_find_merges, the merge queue, close_for with
// merged ids) and its session notify_at (SjNotifyAt), K9's store reservation, compaction, ordering and placement.
// Unordered: k_scwin_apply, one thread per key, runs the late test, plays the on-time values in arrival order, merges
// and closes.  Ordered: k_scwin_apply runs the late test and fills K8's pool; K8's sort puts the due entries in play
// order; k_scwin_flush, one thread per slot, plays them, carries the rest over, merges and closes.  Notify and EOF mark
// the keys with K8's k_jwin_mark and run the same flush.
//
// Playing a value appends ONE entry to the store: the session's cell, the value's rank in the session's list, the
// handle.  A merge of B into A, when the merge queue applies it, records on B's cell the cell that now holds its values
// (A's) and where B's list starts in A's list (A's count then), and adds B's count to A's; A gains the interval
// [base, base + B.cnt) and B's own intervals shifted by base.  A chain C -> B -> A within one call resolves to A's cell
// and the summed base at once, so no thread ever copies a list: a merge costs its key's thread O(M) and the gather O(1)
// per entry.
// Intervals of one session are nested or disjoint (a tree); by (start ascending, end descending) they are its pre-order.
//
// k_scwin_gather, over the whole store, after the per-key kernels of every call that merged or closed: an entry of a
// cell merged away in this call is retagged to the root's cell, rank + base; an entry whose (root) session closed in this
// call moves to the closed record's staging range at its rank, is dead, and releases its handle (a value belongs to
// exactly one session, so the "highest window" bit of K9's entries is always set).  A cell merged away in a call is free
// again only after that call's gather: the walk never reuses a cell of a record it holds, live or merged away.
//
// Handles: a value's is released by its entry in the call that closes its session, a late item's in the call that
// received it.  Session state is never discarded (:798-806), so the clock outlives the sessions.
//
// Per key (slot), never freed:
//   keys[slot], st[slot]     as K8 (JwTable; its JwWin array is not used)
//   kx[slot]                 next session id, held merged ids, held intervals
//   rec[slot * M ...]        sessions (id, open, close, count, cell) in id order == the reference's dict order
//   mrg[slot * 2M ...]       (owner id, merged id) pairs, the `merged_ids` sets of the live sessions (K10)
//   iv[slot * M ...]         (owner id, start, end): the merge intervals of the live sessions, transitive ones included
// Per cell (slot * M + cell): K9's cell_ord / cell_c (the call in which the session on the cell closed, its record) and
//   cell_mord / cell_root / cell_base (the call in which it was merged away, the cell that finally took its values, and
//   where its list starts there).
#pragma once
#include "../../include/bwgpu.h"
#include "bw_collect.cuh"
#include "bw_session.cuh"
#include "bw_sjwin.cuh"

struct __align__(16) ScRec {
  i64 id, open, close;
  u32 cnt;   // values in the session's list, merged ones included
  u32 cell;
};
struct ScIv {
  i64 owner;  // the live session whose list holds [lo, hi) as one merged-away session's values
  u32 lo, hi;
};
struct ScKey {
  i64 next_id;  // max_key + 1 (never resets)
  u32 nm, ni;   // held merged ids, held intervals
};
struct ScTable : CwTable {  // K9's keys, clock / queue state, cells, error words (its window records are not used)
  ScRec* rec;
  ScKey* kx;
  i64* mrg;
  ScIv* iv;
  u64* cell_mord;
  u64* cell_root;
  u32* cell_base;
  i64 gap;
};
struct ScEmit : CwEmit {  // K9's closed records, late rows (window id LATE_SESSION_ID), releases, carry-over, staging
  // per closed record: the session's bounds, its merged ids [moff, moff + mcnt) and intervals [ioff, ioff + icnt)
  i64 *open, *close;
  u64 *moff, *mcnt, *ioff, *icnt;
  i64* mids;
  u64* ivs;  // (start << 32) | end
  unsigned long long *n_mids, *n_ivs;
  unsigned long long* n_mrg;  // merges applied so far (the gather runs after a call that merged)
};

// a late item: one row, window LATE_SESSION_ID (windowing.py:764-766, :1125-1127), naming input row o
__device__ __forceinline__ void bw_sc_late_row(const ScTable& t, const ScEmit& e, const JwParams& p, u64 key, u32 o, u64& lseq) {
  const u64 i = atomicAdd(e.n_late, 1ULL);
  if (i >= e.max_late) {
    bw_jw_fail(t, BW_JW_FULL_LATE);
    return;
  }
  e.l_key[i] = key;
  e.l_wid[i] = (u64)BW_SESS_LATE_ID;
  e.l_epoch[i] = p.epoch;
  e.l_act[i] = p.batch_no;
  e.l_row[i] = o;
  e.l_ord[i] = p.ord;
  e.l_seq[i] = lseq++;
}

// one due value: open_for (K10's walk), then the folder on the session it returned, even one its own find_merges just
// took away (windowing.py:1064-1077): the value's entry goes to es[ei++]; false when the key needs more than M records
// or merged ids
__device__ bool bw_sc_play(const ScTable& t, const CwStore& es, u64 slot, ScRec* R, i64* MG, SessWalk& w, unsigned char* qo,
                           unsigned char* qt, ScKey& kx, i64 ts, u64 h, u64& ei) {
  const u32 M = (u32)t.j.M;
  bool fresh;
  const int i = bw_sess_open_for(R, MG, w, qo, qt, (int)M, t.gap, ts, fresh);
  if (i < 0) return false;
  ScRec& r = R[i];
  if (fresh) {  // a new session, id max_key + 1, on the lowest cell no record the key holds has
    u64 used = 0;
    for (u32 k = 0; k + 1 < w.n; ++k) used |= 1ULL << R[k].cell;
    r.id = kx.next_id++;
    r.open = r.close = ts;
    r.cnt = 0;
    r.cell = (u32)__ffsll((long long)~used) - 1;
  }
  es.ref[ei] = ((slot * M + r.cell) << 1) | 1ULL;
  es.rank[ei] = r.cnt++;
  es.h[ei] = h;
  ++ei;
  return true;
}

// the nv intervals of session `id`, by (start ascending, end descending): each pass writes the smallest key above the
// previous one (a session's intervals are distinct)
__device__ __forceinline__ void bw_sc_ivs(const ScIv* IV, u32 ni, i64 id, u32 nv, u64* out) {
  u64 prev = 0;
  for (u32 c = 0; c < nv; ++c) {
    u64 best = ~0ULL;
    for (u32 k = 0; k < ni; ++k) {
      const u64 sk = ((u64)IV[k].lo << 32) | (0xffffffffu - IV[k].hi);
      if (IV[k].owner == id && (c == 0 || sk > prev) && sk < best) best = sk;
    }
    out[c] = (best & 0xffffffff00000000ULL) | (0xffffffffu - (u32)best);
    prev = best;
  }
}

// `_handle_merged` (windowing.py:1079-1085) with the merger, then `_handle_closed` (:1087-1093) at watermark wm: a record
// and a staging range per closing session, in id order.  False when the key's live sessions would hold more than M
// intervals.
__device__ bool bw_sc_finish(const ScTable& t, const ScEmit& e, const JwParams& p, u64 key, u64 slot, ScRec* R, i64* MG, ScIv* IV,
                             SessWalk& w, const unsigned char* qo, const unsigned char* qt, ScKey& kx, i64 wm) {
  const u32 M = (u32)t.j.M;
  const u64 c0 = slot * M;
  u64 moved = 0;  // cells merged away in this call
  bool full = false;
  bw_sess_merge_each(R, w, qo, qt, [&](ScRec& into, const ScRec& orig) {
    // what merged into orig earlier in this call lies in into's list now, behind into's values
    for (u64 m = moved; m; m &= m - 1) {
      const u64 c = c0 + (u64)(__ffsll((long long)m) - 1);
      if (t.cell_root[c] == c0 + orig.cell) {
        t.cell_root[c] = c0 + into.cell;
        t.cell_base[c] += into.cnt;
      }
    }
    const u64 oc = c0 + orig.cell;
    t.cell_root[oc] = c0 + into.cell;
    t.cell_base[oc] = into.cnt;
    t.cell_mord[oc] = p.ord;
    moved |= 1ULL << orig.cell;
    for (u32 k = 0; k < kx.ni; ++k)
      if (IV[k].owner == orig.id) {
        IV[k].owner = into.id;
        IV[k].lo += into.cnt;
        IV[k].hi += into.cnt;
      }
    if (kx.ni >= M) {
      full = true;
    } else {
      IV[kx.ni].owner = into.id;
      IV[kx.ni].lo = into.cnt;
      IV[kx.ni].hi = into.cnt + orig.cnt;
      ++kx.ni;
    }
    into.cnt += orig.cnt;
  });
  if (full) return false;
  if (moved) atomicAdd(e.n_mrg, 1ULL);
  u64 seq = 0;
  bw_sess_close_each(R, MG, w.n, w.nm, bw_sess_close_after(wm, t.gap), [&](const ScRec& r, u32 cnt) {
    u32 nv = 0;
    for (u32 k = 0; k < kx.ni; ++k) nv += IV[k].owner == r.id;
    const u64 c = atomicAdd(e.n_rows, 1ULL);
    const u64 m0 = cnt ? atomicAdd(e.n_mids, (unsigned long long)cnt) : 0;
    const u64 v0 = nv ? atomicAdd(e.n_ivs, (unsigned long long)nv) : 0;
    if (c >= e.max_rows || m0 + cnt > e.max_rows || v0 + nv > e.max_rows) {
      bw_jw_fail(t, BW_JW_FULL_EMIT);
    } else {
      const u64 at = atomicAdd(e.n_stage, (unsigned long long)r.cnt);
      if (at + r.cnt > e.max_stage) {  // (sized by the host for every entry held: never reached)
        bw_jw_fail(t, BW_CW_FULL_STORE);
      } else {
        e.key[c] = key;
        e.wid[c] = (u64)r.id;
        e.cnt[c] = r.cnt;
        e.soff[c] = at;
        e.epoch[c] = p.epoch;
        e.ord[c] = p.ord;
        e.seq[c] = seq++;
        e.open[c] = r.open;
        e.close[c] = r.close;
        e.moff[c] = m0;
        e.mcnt[c] = cnt;
        e.ioff[c] = v0;
        e.icnt[c] = nv;
        bw_sess_mids(MG, w.nm, r.id, cnt, e.mids + m0);
        bw_sc_ivs(IV, kx.ni, r.id, nv, e.ivs + v0);
        t.cell_c[c0 + r.cell] = c;
        t.cell_ord[c0 + r.cell] = p.ord;
      }
    }
    u32 k = 0;  // its intervals go with it
    for (u32 j = 0; j < kx.ni; ++j)
      if (IV[j].owner != r.id) IV[k++] = IV[j];
    kx.ni = k;
  });
  kx.nm = w.nm;
  return true;
}

// pass A, one thread per key segment: K8's late test per item; unordered, then the play of the on-time items in arrival
// order, the merges and the close; ordered, the on-time items go to K8's pool at base + q
__global__ void k_scwin_apply(ScTable t, ScEmit e, CwStore es, JwParams p, JwPool pool, u64 base, const u64* ksorted, const u32* isorted,
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
    bw_jw_begin(st, p);  // (kx starts at zero: k_scwin_init)
    u64 end = h;
    while (end < n && ksorted[end] == key) ++end;
    i64 wm = BW_UTC_MIN_US;
    u64 lseq = 0, entries = 0;
    for (u64 q = h; q < end; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      const bool is_late = bw_jw_on_item(st, p, ts, wm);
      if (is_late) {
        bw_sc_late_row(t, e, p, key, o, lseq);
        bw_jw_release(t, e, handles[o]);
      } else {
        ++entries;
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
      ScRec* R = t.rec + s * (u64)t.j.M;
      i64* MG = t.mrg + s * (u64)(2 * t.j.M);
      ScKey kx = t.kx[s];
      unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
      SessWalk w;
      bw_sess_walk_begin(w, st.n, kx.nm);
      bool full = false;
      for (u64 q = h; q < end && !full; ++q) {
        if (late[q]) continue;
        const u32 o = isorted[q];
        full = !bw_sc_play(t, es, s, R, MG, w, qo, qt, kx, ts_us[o], handles[o], ei);
      }
      if (full || !bw_sc_finish(t, e, p, key, s, R, MG, t.iv + s * (u64)t.j.M, w, qo, qt, kx, wm)) {
        bw_cw_kill(es, ei, eend);
        bw_jw_fail(t, BW_JW_FULL_WINDOWS);
        continue;  // the call fails and the collect refuses further work: no row of this key is emitted half-done
      }
      st.n = w.n;
      t.kx[s] = kx;
    }
    t.j.st[s] = st;
  }
}

// pass B, one thread per slot: a woken key plays its due entries (in ts order, ties in arrival order), keeps the others
// queued in arrival order, merges and closes; an idle key's entries move to the next pool unchanged.  Also the notify /
// EOF flush of unordered mode (perm NULL: nothing queued).
__global__ void k_scwin_flush(ScTable t, ScEmit e, CwStore es, JwParams p, JwPool pool, const u32* perm) {
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
    if (!bw_cw_reserve(t, es, entries, ei)) continue;
    const u64 eend = ei + entries;
    ScRec* R = t.rec + s * (u64)t.j.M;
    i64* MG = t.mrg + s * (u64)(2 * t.j.M);
    ScKey kx = t.kx[s];
    unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];
    SessWalk w;
    bw_sess_walk_begin(w, st.n, kx.nm);
    bool full = false;
    for (u32 i = qb; i < qe && !full; ++i) {
      const u32 x = perm[i];
      if (pool.side[x] != BW_JW_DROP && woken && pool.ts[x] <= st.wm) full = !bw_sc_play(t, es, s, R, MG, w, qo, qt, kx, pool.ts[x], pool.h[x], ei);
    }
    if (full || (woken && !bw_sc_finish(t, e, p, t.j.keys[s], s, R, MG, t.iv + s * (u64)t.j.M, w, qo, qt, kx, st.wm))) {
      bw_cw_kill(es, ei, eend);
      bw_jw_fail(t, BW_JW_FULL_WINDOWS);
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

// after the per-key kernels of a call that merged or closed (rows0 / mrg0: the record and merge counts before it): every
// entry of a cell merged away in this call is retagged to the cell that took its values; every entry whose session closed
// in this call goes to its record's staging range at its rank, is dead, and releases its handle
__global__ void k_scwin_gather(ScTable t, ScEmit e, CwStore es, JwParams p, u64 rows0, u64 mrg0) {
  if (*e.n_rows == rows0 && *e.n_mrg == mrg0) return;
  const u64 n = *es.n;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  for (u64 b = (u64)blockIdx.x * blockDim.x; b < n; b += stride) {  // (b is warp-uniform: the whole warp reaches the ballot)
    const u64 i = b + threadIdx.x;
    bool rel = false;
    u64 h = 0;
    if (i < n) {
      const u64 r = es.ref[i];
      if (r != BW_CW_DEAD) {
        u64 c = r >> 1;
        u32 rank = es.rank[i];
        const bool moved = t.cell_mord[c] == p.ord;
        if (moved) {
          rank += t.cell_base[c];
          c = t.cell_root[c];
        }
        if (t.cell_ord[c] == p.ord) {
          const u64 rc = t.cell_c[c];
          const u64 j = e.soff[rc] + rank;
          h = es.h[i];
          e.stage[j] = h;
          e.stage_rec[j] = (u32)rc;
          es.ref[i] = BW_CW_DEAD;
          rel = true;
        } else if (moved) {
          es.ref[i] = (c << 1) | 1ULL;
          es.rank[i] = rank;
        }
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

__global__ void k_scwin_init(ScTable t) {
  const u64 cells = (t.j.cap + 1) * (u64)t.j.M;
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < cells; s += (u64)gridDim.x * blockDim.x) {
    t.cell_ord[s] = ~0ULL;
    t.cell_mord[s] = ~0ULL;
    if (s > t.j.cap) continue;
    t.j.keys[s] = BW_EMPTY_KEY;
    t.j.st[s].init = 0;
    t.j.st[s].n = t.j.st[s].nq = 0;
    t.j.st[s].qord = ~0ULL;
    t.j.st[s].act = ~0ULL;
    t.kx[s].next_id = 0;
    t.kx[s].nm = t.kx[s].ni = 0;
  }
}
