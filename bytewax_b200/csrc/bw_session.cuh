// bw_session.cuh -- K7: session-window folds (count / sum / min / max) over `SessionWindower`.
//
// The reference runs `_WindowLogic.on_batch` over `_SessionWindowerLogic` (pysrc/bytewax/operators/windowing.py:
// 1115-1133, 671-810): one Python `open_for` / `_session_find_merges` call per item, per key in arrival order.
// Sessions are order-dependent -- ids are per-key counters, the first matching session by id wins, merges happen as
// they are found -- so the device does what K6 does: group the activation by key (CUB stable sort, `keyed_group`),
// then ONE thread walks each key's items in arrival order and restates the reference step by step.  Each value is
// folded in the reference's own order, so every accumulator is bit-identical to it (i64 sums wrap past 2^63).
//
// A hot key is walked serially while the rest of the grid idles: every item scans the key's n held sessions, and every
// item that extends one re-sorts them by open time (insertion sort), so up to O(items x n^2), n <= max_sessions_per_key.
//
// Per key, never freed (session state is never discarded, windowing.py:798-806):
//   keys[slot]                 the key (bw_keyed_find table; slot `cap` is the BW_EMPTY_KEY alias slot)
//   st[slot]                   next session id, the EventClock pair (watermark_base, system time of max event),
//                              live sessions n, held merged ids nm
//   rec[slot * M ...]          sessions (id, open, close, acc) in id order == the reference's dict order
//   mrg[slot * 2M ...]         (owner id, merged id) pairs, the `merged_ids` sets of the live sessions
#pragma once
#include "../../include/bwgpu.h"
#include "bw_common.cuh"
#include "bw_keyed.cuh"

#define BW_SESS_MAXM 64
#define BW_SESS_LATE_ID (-1LL)  // LATE_SESSION_ID, windowing.py:671
// reasons behind a BW_ERR_CAPACITY, or-ed into SessTable::why
enum { BW_SESS_FULL_TABLE = 1, BW_SESS_FULL_SESSIONS = 2, BW_SESS_FULL_EMIT = 4, BW_SESS_FULL_LATE = 8, BW_SESS_FULL_MERGED = 16 };

struct SessState {
  i64 next_id;   // max_key + 1
  i64 wm_base;   // _EventClockState.watermark_base
  i64 sys_max;   // _EventClockState.system_time_of_max_event
  u32 n, nm;     // live sessions, held merged ids
  u32 init, pad;
};
struct __align__(32) SessRec {
  i64 id, open, close;
  u64 acc;
};
struct SessTable {
  u64* keys;
  SessState* st;
  SessRec* rec;
  i64* mrg;
  u64 cap;
  int M;
  u32* err;  // BW_ERR_CAPACITY once anything overflowed
  u32* why;  // BW_SESS_FULL_* bits
};
struct SessEmit {
  // closed sessions
  u64* key;
  i64* wid;
  u64* acc;
  i64 *open, *close;
  u64 *epoch, *ord, *moff, *mcnt;
  u64 max_rows;
  unsigned long long* n_rows;
  i64* mids;  // merged ids of the closed rows, [moff, moff + mcnt) per row
  unsigned long long* n_mids;
  // late items
  u64 *l_key, *l_epoch, *l_ord, *l_act, *l_row;
  u64 max_late;
  unsigned long long* n_late;
};
struct SessParams {
  int red, is_f64;
  i64 gap, wait, now;
  u64 epoch, ord;
  u32 batch_no;
};

__device__ __forceinline__ void bw_sess_fail(const SessTable& t, u32 bit) {
  atomicOr(t.why, bit);
  atomicCAS(t.err, 0u, (u32)BW_ERR_CAPACITY);
}

// `folder(acc, v)`: count `acc + 1`, reduce_window's `operator.add`, `max(acc, v)` / `min(acc, v)` (the first argument
// stays unless the second is strictly greater / less)
__device__ __forceinline__ u64 bw_sess_combine(int red, int is_f64, u64 a, u64 b) {
  if (red == BW_RED_SUM) return is_f64 ? (u64)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b))) : a + b;
  bool take;
  if (is_f64) {
    const double x = __longlong_as_double((long long)a), y = __longlong_as_double((long long)b);
    take = red == BW_RED_MAX ? (y > x) : (y < x);
  } else {
    take = red == BW_RED_MAX ? ((i64)b > (i64)a) : ((i64)b < (i64)a);
  }
  return take ? b : a;
}
__device__ __forceinline__ u64 bw_sess_fold(const SessParams& p, u64 acc, u64 v) {
  return p.red == BW_RED_COUNT ? acc + 1 : bw_sess_combine(p.red, p.is_f64, acc, v);
}
// merger(into, orig), windowing.py:1700-1703: count `into + orig`, the reducer otherwise
__device__ __forceinline__ u64 bw_sess_merge(const SessParams& p, u64 into, u64 orig) {
  return p.red == BW_RED_COUNT ? into + orig : bw_sess_combine(p.red, p.is_f64, into, orig);
}

// ---- the per-key session steps: K10 (bw_sjwin.cuh) walks with all of them, K7 closes and notifies with them -----------
// R: a session record with `id`, `open` and `close` (SessRec here, SjRec there); MG: the key's (owner id, merged id)
// pairs.  One thread walks a key; the walk of one call's inserts is SessWalk.
// (scalars only, so they stay in registers; the merge queue, (orig, into) record indices in discovery order, lives in
// the caller's local arrays qo / qt of BW_SESS_MAXM entries, passed to the steps that use it)
struct SessWalk {
  u32 n, nm;  // records held (live, or merged away in this call), held merged ids
  u32 nq;     // merge queue entries
  u64 dead;   // records merged away in this call (bit i = R[i])
};
__device__ __forceinline__ void bw_sess_walk_begin(SessWalk& w, u32 n, u32 nm) {
  w.n = n;
  w.nm = nm;
  w.nq = 0;
  w.dead = 0;
}

// _session_find_merges, windowing.py:688-715: live records stably sorted by open (ties keep id order), each merged into
// the running survivor when it opens within gap of the survivor's close; false when the survivors would hold more than
// M merged ids
template <class R>
__device__ __forceinline__ bool bw_sess_find_merges(R* Rs, i64* MG, SessWalk& w, unsigned char* qo, unsigned char* qt, int M, i64 gap) {
  unsigned char ix[BW_SESS_MAXM];
  u32 nl = 0;
  for (u32 i = 0; i < w.n; ++i)
    if (!(w.dead >> i & 1)) {
      u32 j = nl++;
      const i64 op = Rs[i].open;
      while (j > 0 && Rs[ix[j - 1]].open > op) {
        ix[j] = ix[j - 1];
        --j;
      }
      ix[j] = (unsigned char)i;
    }
  if (nl < 2) return true;
  u32 last = ix[0];
  for (u32 j = 1; j < nl; ++j) {
    const u32 th = ix[j];
    if (Rs[th].open - Rs[last].close <= gap) {
      if (Rs[th].close > Rs[last].close) Rs[last].close = Rs[th].close;
      w.dead |= 1ULL << th;
      qo[w.nq] = (unsigned char)th;
      qt[w.nq] = (unsigned char)last;
      ++w.nq;
      const i64 gone = Rs[th].id;  // its own merged ids go with it; the survivor gains its id
      u32 k = 0;
      for (u32 m = 0; m < w.nm; ++m)
        if (MG[2 * m] != gone) {
          MG[2 * k] = MG[2 * m];
          MG[2 * k + 1] = MG[2 * m + 1];
          ++k;
        }
      w.nm = k;
      if (w.nm >= (u32)M) return false;
      MG[2 * w.nm] = Rs[last].id;
      MG[2 * w.nm + 1] = gone;
      ++w.nm;
    } else {
      last = th;
    }
  }
  return true;
}

// open_for, windowing.py:731-762: the first live session by id that takes the timestamp (merging after an extension).
// The index the value goes to -- even if a merge just took that session away (windowing.py:1069-1076) -- or, with
// `fresh` set, the index of a new record the caller opens there (id max_key + 1, open = close = ts); -1 when the key
// needs more than M records or merged ids.
template <class R>
__device__ __forceinline__ int bw_sess_open_for(R* Rs, i64* MG, SessWalk& w, unsigned char* qo, unsigned char* qt, int M, i64 gap, i64 ts,
                                                 bool& fresh) {
  fresh = false;
  int hit = -1;
  bool moved = false;
  for (u32 i = 0; i < w.n; ++i) {
    if (w.dead >> i & 1) continue;
    const i64 op = Rs[i].open, cl = Rs[i].close;
    if (op <= ts && ts <= cl) {
      hit = (int)i;
      break;
    }
    if (op - ts > 0 && op - ts <= gap) {
      Rs[i].open = ts;
      hit = (int)i;
      moved = true;
      break;
    }
    if (ts - cl > 0 && ts - cl <= gap) {
      Rs[i].close = ts;
      hit = (int)i;
      moved = true;
      break;
    }
  }
  if (moved) return bw_sess_find_merges(Rs, MG, w, qo, qt, M, gap) ? hit : -1;
  if (hit >= 0) return hit;
  if (w.n >= (u32)M) return -1;
  fresh = true;
  return (int)w.n++;
}

// _handle_merged, windowing.py:1079-1085: `on_merge(into, orig)` in discovery order, then the merged-away records leave
template <class R, class F>
__device__ __forceinline__ void bw_sess_merge_each(R* Rs, SessWalk& w, const unsigned char* qo, const unsigned char* qt, F&& on_merge) {
  for (u32 j = 0; j < w.nq; ++j) on_merge(Rs[qt[j]], Rs[qo[j]]);
  u32 k = 0;
  for (u32 i = 0; i < w.n; ++i)
    if (!(w.dead >> i & 1)) Rs[k++] = Rs[i];
  w.n = k;
  w.nq = 0;
  w.dead = 0;
}

// close_for (windowing.py:774-788): live sessions with close < close_after leave in id order; `on_close(r, cnt)` sees
// each while its cnt merged ids are still in MG (bw_sess_mids writes them), then they go with it
template <class R, class F>
__device__ __forceinline__ void bw_sess_close_each(R* Rs, i64* MG, u32& n, u32& nm, i64 close_after, F&& on_close) {
  u32 w = 0;
  for (u32 i = 0; i < n; ++i) {
    const R r = Rs[i];
    if (!(r.close < close_after)) {
      Rs[w++] = r;
      continue;
    }
    u32 cnt = 0;
    for (u32 j = 0; j < nm; ++j) cnt += MG[2 * j] == r.id;
    on_close(r, cnt);
    u32 k = 0;
    for (u32 j = 0; j < nm; ++j)
      if (MG[2 * j] != r.id) {
        MG[2 * k] = MG[2 * j];
        MG[2 * k + 1] = MG[2 * j + 1];
        ++k;
      }
    nm = k;
  }
  n = w;
}

// the cnt merged ids of session `id`, ascending: each pass writes the smallest id above the previous one (ids are distinct)
__device__ __forceinline__ void bw_sess_mids(const i64* MG, u32 nm, i64 id, u32 cnt, i64* out) {
  i64 prev = -1;
  for (u32 c = 0; c < cnt; ++c) {
    i64 best = INT64_MAX;
    for (u32 j = 0; j < nm; ++j)
      if (MG[2 * j] == id && MG[2 * j + 1] > prev && MG[2 * j + 1] < best) best = MG[2 * j + 1];
    out[c] = best;
    prev = best;
  }
}

__device__ __forceinline__ i64 bw_sess_close_after(i64 watermark, i64 gap) {
  const i64 c = watermark - gap;  // watermark >= UTC_MIN and gap <= UTC_MAX - UTC_MIN: no overflow
  return c < BW_UTC_MIN_US ? BW_UTC_MIN_US : c;
}

// notify_at of the session windower (windowing.py:790-796) is min(close) + gap: true when it has come by `now`
template <class R>
__device__ __forceinline__ bool bw_sess_due(const R* Rs, u32 n, i64 gap, i64 now) {
  if (n == 0) return false;
  i64 mc = Rs[0].close;
  for (u32 i = 1; i < n; ++i) mc = Rs[i].close < mc ? Rs[i].close : mc;
  return mc <= now - gap;
}

// ---- K7 --------------------------------------------------------------------------------------------------------------
// close_for with K7's rows: E + M rows, merged ids ascending
__device__ void bw_sess_close(const SessTable& t, const SessEmit& e, u64 key, SessRec* R, i64* MG, u32& n, u32& nm, i64 close_after,
                              u64 epoch, u64 ord) {
  bw_sess_close_each(R, MG, n, nm, close_after, [&](const SessRec& r, u32 cnt) {
    const u64 row = atomicAdd(e.n_rows, 1ULL);
    const u64 m0 = cnt ? atomicAdd(e.n_mids, (unsigned long long)cnt) : 0;
    if (row >= e.max_rows || m0 + cnt > e.max_rows) {
      bw_sess_fail(t, BW_SESS_FULL_EMIT);
      return;
    }
    e.key[row] = key;
    e.wid[row] = r.id;
    e.acc[row] = r.acc;
    e.open[row] = r.open;
    e.close[row] = r.close;
    e.epoch[row] = epoch;
    e.ord[row] = ord;
    e.moff[row] = m0;
    e.mcnt[row] = cnt;
    bw_sess_mids(MG, nm, r.id, cnt, e.mids + m0);
  });
}

// one thread per key segment: the key's items of this activation in arrival order.  The walk restates open_for and
// _session_find_merges inline rather than through bw_sess_open_for / bw_sess_merge_each: routed through them, this kernel
// compiled to a different layout and ran ~5% slower in tools/bench_sessions.py on an H100 80GB HBM3 at a 700 W power
// limit (5.34 vs 5.08 ms per activation, three alternating runs each).  The two must agree; K10's goldens and K7's both
// pin them to the reference.
__global__ void k_session_apply(SessTable t, SessEmit e, SessParams p, const u64* ksorted, const u32* isorted, const u32* headpos,
                                const u64* vals, const i64* ts_us, u64 n) {
  const int M = t.M;
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.keys, t.cap, key, t.err);
    if (s == ~0ULL) {
      bw_sess_fail(t, BW_SESS_FULL_TABLE);
      continue;
    }
    SessState st = t.st[s];
    if (!st.init) {  // builder(None): _EventClockLogic.__post_init__ (windowing.py:245-248), empty windower state
      st.init = 1;
      st.next_id = 0;
      st.wm_base = BW_UTC_MIN_US;
      st.sys_max = p.now;
      st.n = st.nm = 0;
    }
    SessRec* R = t.rec + s * (u64)M;
    i64* MG = t.mrg + s * (u64)(2 * M);
    u32 n_rec = st.n, nm = st.nm;  // n_rec: records held, live or merged away in this activation
    u64 dead = 0;                  // records merged away in this activation (bit i = R[i])
    unsigned char qo[BW_SESS_MAXM], qt[BW_SESS_MAXM];  // merge queue: (orig, into) record indices in discovery order
    u32 nq = 0;
    bool full = false;
    i64 wm = BW_UTC_MIN_US;
    for (u64 q = h; q < n && ksorted[q] == key && !full; ++q) {
      const u32 o = isorted[q];
      const i64 ts = ts_us[o];
      // _EventClockLogic.on_item, windowing.py:263-287 (ts - wait below UTC_MIN raises OverflowError: ignored)
      wm = st.wm_base + (p.now - st.sys_max);
      if (p.wait != BW_WAIT_FOREVER && ts - BW_UTC_MIN_US >= p.wait) {
        const i64 cand = ts - p.wait;
        if (cand > wm) {
          st.wm_base = cand;
          st.sys_max = p.now;
          wm = cand;
        }
      }
      if (ts < wm) {  // late: one row, window LATE_SESSION_ID (windowing.py:1125-1127, 764-766)
        const u64 i = atomicAdd(e.n_late, 1ULL);
        if (i >= e.max_late) {
          bw_sess_fail(t, BW_SESS_FULL_LATE);
        } else {
          e.l_key[i] = key;
          e.l_epoch[i] = p.epoch;
          e.l_ord[i] = p.ord;
          e.l_act[i] = p.batch_no;
          e.l_row[i] = o;
        }
        continue;
      }
      const u64 v = vals ? vals[o] : 0;
      // open_for, windowing.py:731-762: the first live session by id that takes the timestamp
      int hit = -1;
      bool moved = false;
      for (u32 i = 0; i < n_rec; ++i) {
        if (dead >> i & 1) continue;
        const i64 op = R[i].open, cl = R[i].close;
        if (op <= ts && ts <= cl) {
          hit = (int)i;
          break;
        }
        if (op - ts > 0 && op - ts <= p.gap) {
          R[i].open = ts;
          hit = (int)i;
          moved = true;
          break;
        }
        if (ts - cl > 0 && ts - cl <= p.gap) {
          R[i].close = ts;
          hit = (int)i;
          moved = true;
          break;
        }
      }
      if (moved) {
        // _session_find_merges, windowing.py:688-715: live records stably sorted by open (ties keep id order), each
        // merged into the running survivor when it opens within gap of the survivor's close
        unsigned char ix[BW_SESS_MAXM];
        u32 nl = 0;
        for (u32 i = 0; i < n_rec; ++i)
          if (!(dead >> i & 1)) {
            u32 j = nl++;
            const i64 op = R[i].open;
            while (j > 0 && R[ix[j - 1]].open > op) {
              ix[j] = ix[j - 1];
              --j;
            }
            ix[j] = (unsigned char)i;
          }
        if (nl >= 2) {
          u32 last = ix[0];
          for (u32 j = 1; j < nl; ++j) {
            const u32 th = ix[j];
            if (R[th].open - R[last].close <= p.gap) {
              if (R[th].close > R[last].close) R[last].close = R[th].close;
              dead |= 1ULL << th;
              qo[nq] = (unsigned char)th;
              qt[nq] = (unsigned char)last;
              ++nq;
              const i64 gone = R[th].id;  // its own merged ids go with it; the survivor gains its id
              u32 k = 0;
              for (u32 m = 0; m < nm; ++m)
                if (MG[2 * m] != gone) {
                  MG[2 * k] = MG[2 * m];
                  MG[2 * k + 1] = MG[2 * m + 1];
                  ++k;
                }
              nm = k;
              if (nm >= (u32)M) {
                full = true;
                break;
              }
              MG[2 * nm] = R[last].id;
              MG[2 * nm + 1] = gone;
              ++nm;
            } else {
              last = th;
            }
          }
        }
        if (full) break;
      }
      if (hit < 0) {  // a new session, id max_key + 1
        if (n_rec >= (u32)M) {
          full = true;
          break;
        }
        SessRec r;
        r.id = st.next_id++;
        r.open = r.close = ts;
        r.acc = p.red == BW_RED_COUNT ? 1ULL : v;  // builder(None) then the first value
        R[n_rec++] = r;
      } else {
        // the value goes to the id open_for returned, even if a merge just took that session away (windowing.py:1069-1076)
        R[hit].acc = bw_sess_fold(p, R[hit].acc, v);
      }
    }
    if (full) {
      bw_sess_fail(t, BW_SESS_FULL_SESSIONS);
      continue;  // the call fails and the fold refuses further work: no row of this key is emitted half-done
    }
    // _handle_merged, windowing.py:1079-1085: into = merger(into, orig), in discovery order
    for (u32 j = 0; j < nq; ++j) R[qt[j]].acc = bw_sess_merge(p, R[qt[j]].acc, R[qo[j]].acc);
    u32 w = 0;
    for (u32 i = 0; i < n_rec; ++i)
      if (!(dead >> i & 1)) R[w++] = R[i];
    n_rec = w;
    // _handle_closed with the watermark after the key's last item (windowing.py:1132, 1087-1093)
    bw_sess_close(t, e, key, R, MG, n_rec, nm, bw_sess_close_after(wm, p.gap), p.epoch, p.ord);
    st.n = n_rec;
    st.nm = nm;
    t.st[s] = st;
  }
}

// K7 on world > 1, at the owner: the received segments (bv.h_counts rows from each source) into K7's columns in (source
// rank, source order), the arrival order a world-1 fold sees when it is fed the rank-major concatenation.  name[i] =
// source rank << 32 | the row's index in that source's columns (src_row: the region's row column, `cap` rows per source).
// vals is NULL for count, which sends none.
__global__ void k_xsess_gather(BatchView bv, const u32* src_row, u64 cap, u64 n, u64* keys, u64* vals, i64* ts, u64* name) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    int r = 0;
    u64 o = i;
    while (o >= bv.h_counts[r]) o -= bv.h_counts[r++];
    keys[i] = bv.keys[r][o];
    if (vals) vals[i] = ((const u64*)bv.vals[r])[o];
    ts[i] = bv.ts[r][o];
    name[i] = (u64)r << 32 | src_row[(u64)r * cap + o];
  }
}

// After k_session_apply on world > 1: the late rows this call added, [*before, min(*n_late, max_late)), hold positions in
// the gathered columns; give them their rows' names instead.  Names grow with the position, so arrival order holds.
__global__ void k_xsess_name_late(const unsigned long long* before, const unsigned long long* n_late, u64 max_late, u64* l_row,
                                  const u64* name) {
  const u64 hi = *n_late < max_late ? *n_late : max_late;
  for (u64 i = *before + (u64)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (u64)gridDim.x * blockDim.x) l_row[i] = name[l_row[i]];
}

// notify phase (src/operators.rs:808-858): a key is due when min(close) + gap <= now (`notify_at`, windowing.py:790-796,
// identity `to_system_utc`); it closes what its watermark at `now` allows (`on_notify`, :1135-1142, :289-298).
// eof (src/operators.rs:862-894, windowing.py:1144-1151): every key, watermark UTC_MAX.
__global__ void k_session_close_all(SessTable t, SessEmit e, SessParams p, int eof) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    SessState st = t.st[s];
    if (!st.init || st.n == 0) continue;
    SessRec* R = t.rec + s * (u64)t.M;
    i64 wm = BW_UTC_MAX_US;
    if (!eof) {
      if (!bw_sess_due(R, st.n, p.gap, p.now)) continue;
      wm = st.wm_base + (p.now - st.sys_max);
    }
    u32 n_rec = st.n, nm = st.nm;
    bw_sess_close(t, e, t.keys[s], R, t.mrg + s * (u64)(2 * t.M), n_rec, nm, bw_sess_close_after(wm, p.gap), p.epoch, p.ord);
    t.st[s].n = n_rec;
    t.st[s].nm = nm;
  }
}

__global__ void k_session_init(SessTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.keys[s] = BW_EMPTY_KEY;
    t.st[s].init = 0;
    t.st[s].n = t.st[s].nm = 0;
  }
}
