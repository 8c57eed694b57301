// bw_kjoin.cuh -- K15: the window-free keyed `op.join` with 1 to 4 sides: product inserts, and first / last inserts
// with 1, 3 or 4 sides (K6, bw_keyed.cuh, keeps the two-sided first / last join).
//
// The reference runs `_JoinLogic` + `_JoinState` (pysrc/bytewax/operators/__init__.py:2076-2190) under
// `_StatefulLogic.on_batch` (:1030-1042) over the `(key, (side, value))` stream of `_join_label_merge`.  Per key and
// item: "product" appends the value to the side's list (`add_val`), "last" replaces the list with [value] (`set_val`),
// "first" sets it only while the list is empty; "complete" emits `astuples()` once every side is non-empty and discards
// the logic (the key's next item, even in the same batch, starts from empty lists); "running" emits after every item;
// "final" emits at EOF for every key that still has a logic.  `astuples()` is the `itertools.product` of the lists, the
// last side varying fastest, an empty side giving one None.
//
// This is K14 (bw_pjwin.cuh) with one window per key that never closes.  A key's lists are K9's ENTRY STORE
// (bw_collect.cuh): one entry per stored value -- ref = (slot << 2) | side, the value's rank within (key, side), the
// handle.  Per key and side the table keeps the value count and the first rank of the current generation, so a side's
// list is always the ranks [gen, cnt): "last" moves gen up to the new rank, "first" into a non-empty side stores
// nothing, a "complete" emission moves every side's gen up to its cnt.  A side that is empty when a call reaches its key
// restarts its ranks at 0 (all its entries died in earlier calls).
//
// One thread per key (after the stable group-by-key, keyed_group) walks the key's items twice, each item in O(sides)
// work with no list scans: the first walk counts the entries, events, unstored values and dead entries the key adds,
// which it then reserves with one atomic each; the second writes them.  An emission appends an EVENT (key, epoch, call,
// sequence, per side a rank range [lo, hi)); a key that emitted in a call gets one STAGE RECORD covering the union of
// its events' ranges, and k_kjoin_gather copies those entries into staging, over the whole store, so each event can
// still be expanded at advance after later calls moved or compacted the store.  At advance / eof the events are put in
// the reference's order (order_perm: per call, ascending key string, then sequence) and expanded by K14's
// k_pjwin_count, saturating scan and k_pjwin_expand.
//
// Releases: a value has exactly one entry, so the entry's death releases its handle -- a "first" value that was not
// stored in the call that received it (by the walker), a replaced "last" value or an emitted "complete" generation in
// the call that moved gen past it (by the gather, after staging), everything still held at EOF.
#pragma once
#include "../../include/bwgpu.h"
#include "bw_keyed.cuh"
#include "bw_pjwin.cuh"

struct KjCell {
  u32 cnt[BW_JW_MAXSIDES];  // values stored for the side (ranks restart when a call finds the side empty)
  u32 gen[BW_JW_MAXSIDES];  // rank of the first value of the side's current list
};
struct KjTable {
  u64* keys;     // BW_EMPTY_KEY when free; slot `cap` is the alias slot of that key value
  KjCell* cell;
  unsigned char* live;  // the key has a logic (`final` emits these at EOF)
  u64* rec_ord;  // the call in which the key last got a stage record, and its index
  u64* rec_c;
  u64 cap;
  int sides, insert_mode, emit_mode;
  // the fail / release helpers of bw_jwin.cuh read these two
  u32* err;
  u32* why;
};
struct KjEmit {
  // emission events
  u64 *key, *epoch, *ord, *seq, *rec;
  u32 *lo, *hi;  // [event * 4 + side]: the side's list is ranks [lo, hi) of the key
  u64 max_rows;
  unsigned long long* n_rows;
  // released handles
  u64* rel;
  u64 max_rel;
  unsigned long long* n_rel;
  // stage records, one per (key, call) with events: per side the first rank b and the count n staged, and where they
  // start in staging
  u32 *rb, *rn;  // [record * 4 + side]
  u64* rbase;    // [record * 4 + side]
  unsigned long long* n_rec;  // (records <= events: bounded by max_rows)
  u64* stage;
  u64 max_stage;
  unsigned long long* n_stage;
  unsigned long long* n_kill;  // entries whose rank a move of gen passed in this call (the gather runs when some did)
};
struct KjParams {
  u64 epoch, ord;
  int eof;
};
struct KjWalk {  // what one key's items add: store entries, events, values not stored, entries that die
  u64 entries, events, drops, kills;
};

// one event of the key: per side the ranks [gen, cnt); its stage record starts at the first event's gen
__device__ __forceinline__ void bw_kj_event(const KjEmit& e, const KjParams& p, int sides, u64 key, const KjCell& c, u64 row, u64 seq,
                                            u64 rec) {
  e.key[row] = key;
  e.epoch[row] = p.epoch;
  e.ord[row] = p.ord;
  e.seq[row] = seq;
  e.rec[row] = rec;
  for (int s = 0; s < BW_JW_MAXSIDES; ++s) {
    const bool on = s < sides;
    e.lo[row * 4 + s] = on ? c.gen[s] : 0;
    e.hi[row * 4 + s] = on ? c.cnt[s] : 0;
  }
}

// `_StatefulLogic.on_batch` over the key's items [q0, q1) on its state c.  Counting (!WRITE): only w changes, and a
// side >= sides fails the call.  Writing: entries, events and unstored handles go to `at` + their count so far, and
// rb / rn get the key's stage record of this call.  0, or the BW_* reason the key cannot go on.
template <bool WRITE>
__device__ u32 bw_kj_walk(const KjTable& t, const KjEmit& e, const CwStore& es, const KjParams& p, u64 key, u64 slot, KjCell& c, bool& live,
                          KjWalk& w, const KjWalk& at, u64 rec, u32* rb, u32* rn, u64 q0, u64 q1, const u32* isorted, const u64* handles,
                          const unsigned char* sides) {
  const int S = t.sides;
  for (u64 q = q0; q < q1; ++q) {
    const u32 o = isorted[q];
    const int side = sides[o];
    if (side >= S) {  // (device columns are not checked on the host)
      if (!WRITE) {
        atomicOr(t.why, (u32)BW_JW_BAD_SIDE);
        atomicCAS(t.err, 0u, (u32)BW_ERR_SPEC);
      }
      continue;
    }
    live = true;
    if (t.insert_mode == BW_JOIN_INSERT_FIRST && c.cnt[side] != c.gen[side]) {  // `first` into a set side: not stored
      if (WRITE) e.rel[at.drops + w.drops] = handles[o];
      ++w.drops;
    } else {
      if (c.cnt[side] == 0xFFFFFFFFu) return BW_PJ_FULL_SIDE;
      if (WRITE) {
        const u64 i = at.entries + w.entries;
        es.ref[i] = (slot << 2) | (u64)side;
        es.rank[i] = c.cnt[side];
        es.h[i] = handles[o];
      }
      ++w.entries;
      if (t.insert_mode != BW_JOIN_INSERT_PRODUCT) {  // `set_val`: the old list dies
        w.kills += c.cnt[side] - c.gen[side];
        c.gen[side] = c.cnt[side];
      }
      ++c.cnt[side];
    }
    bool emit = t.emit_mode == BW_JOIN_EMIT_RUNNING;
    if (t.emit_mode == BW_JOIN_EMIT_COMPLETE) {
      emit = true;
      for (int s = 0; s < S; ++s) emit = emit && c.cnt[s] > c.gen[s];
    }
    if (!emit) continue;
    if (WRITE) {
      if (w.events == 0)
        for (int s = 0; s < BW_JW_MAXSIDES; ++s) rb[s] = s < S ? c.gen[s] : 0;
      for (int s = 0; s < S; ++s) rn[s] = c.cnt[s] - rb[s];
      bw_kj_event(e, p, S, key, c, at.events + w.events, w.events, rec);
    }
    ++w.events;
    if (t.emit_mode == BW_JOIN_EMIT_COMPLETE) {  // DISCARD: the next item starts from empty lists
      for (int s = 0; s < S; ++s) {
        w.kills += c.cnt[s] - c.gen[s];
        c.gen[s] = c.cnt[s];
      }
      live = false;
    }
  }
  return 0;
}

// the key's stage record `rec` of this call: ranks rb[s] .. rb[s] + rn[s] of each side, and its staging range
__device__ void bw_kj_stage(const KjTable& t, const KjEmit& e, const KjParams& p, u64 slot, u64 rec, const u32* rb, const u32* rn) {
  u64 tot = 0;
  for (int s = 0; s < BW_JW_MAXSIDES; ++s) tot += rn[s];
  u64 at = tot ? atomicAdd(e.n_stage, (unsigned long long)tot) : 0;
  if (at + tot > e.max_stage) {  // (sized by the host for every entry held: never reached)
    bw_jw_fail(t, BW_CW_FULL_STORE);
    return;
  }
  for (int s = 0; s < BW_JW_MAXSIDES; ++s) {
    e.rb[rec * 4 + s] = rb[s];
    e.rn[rec * 4 + s] = rn[s];
    e.rbase[rec * 4 + s] = at;
    at += rn[s];
  }
  t.rec_ord[slot] = p.ord;
  t.rec_c[slot] = rec;
}

// reserve `n` of a buffer's `cap` at *cnt for one key (base in *at); false (and the call fails with `why`) when they do
// not fit
__device__ __forceinline__ bool bw_kj_take(const KjTable& t, unsigned long long* cnt, u64 n, u64 cap, u32 why, u64& at) {
  at = n ? atomicAdd(cnt, (unsigned long long)n) : 0;
  if (at + n <= cap) return true;
  bw_jw_fail(t, why);
  return false;
}

// one thread per key segment: count the key's additions, reserve them, then write them
__global__ void k_kjoin_apply(KjTable t, KjEmit e, CwStore es, KjParams p, const u64* ksorted, const u32* isorted, const u32* headpos,
                              const u64* handles, const unsigned char* sides, u64 n) {
  for (u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (u64)gridDim.x * blockDim.x) {
    if (headpos[h] != h) continue;
    const u64 key = ksorted[h];
    const u64 s = bw_keyed_find(t.keys, t.cap, key, t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      continue;
    }
    u64 end = h + 1;
    while (end < n && ksorted[end] == key) ++end;
    KjCell c = t.cell[s];
    for (int x = 0; x < t.sides; ++x)
      if (c.cnt[x] == c.gen[x]) c.cnt[x] = c.gen[x] = 0;  // an empty side: its entries died in earlier calls
    u32 rb[BW_JW_MAXSIDES] = {0, 0, 0, 0}, rn[BW_JW_MAXSIDES] = {0, 0, 0, 0};
    KjWalk cnt{}, at{};
    bool live = t.live[s];
    {
      KjCell c1 = c;
      bool live1 = live;
      const u32 bad = bw_kj_walk<false>(t, e, es, p, key, s, c1, live1, cnt, at, 0, rb, rn, h, end, isorted, handles, sides);
      if (bad) {
        bw_jw_fail(t, bad);
        continue;  // the call fails and the join refuses further work
      }
    }
    u64 rec = 0;
    if (!bw_kj_take(t, es.n, cnt.entries, es.cap, BW_CW_FULL_STORE, at.entries)) continue;  // (sized by the host: never reached)
    if (!bw_kj_take(t, e.n_rows, cnt.events, e.max_rows, BW_JW_FULL_EMIT, at.events)) continue;
    if (!bw_kj_take(t, e.n_rel, cnt.drops, e.max_rel, BW_JW_FULL_EMIT, at.drops)) continue;  // (sized by the host: never reached)
    if (!bw_kj_take(t, e.n_rec, cnt.events ? 1 : 0, e.max_rows, BW_JW_FULL_EMIT, rec)) continue;
    KjWalk w{};
    bw_kj_walk<true>(t, e, es, p, key, s, c, live, w, at, rec, rb, rn, h, end, isorted, handles, sides);
    t.cell[s] = c;
    t.live[s] = live;
    if (cnt.events) bw_kj_stage(t, e, p, s, rec, rb, rn);
    if (cnt.kills) atomicAdd(e.n_kill, (unsigned long long)cnt.kills);
  }
}

// EOF, one thread per slot: `final` emits every live key's product; every key's lists end (its entries die in the
// gather that follows)
__global__ void k_kjoin_eof(KjTable t, KjEmit e, KjParams p) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    if (!t.live[s]) continue;
    t.live[s] = 0;
    KjCell c = t.cell[s];
    if (t.emit_mode == BW_JOIN_EMIT_FINAL) {
      u64 row, rec;
      if (!bw_kj_take(t, e.n_rows, 1, e.max_rows, BW_JW_FULL_EMIT, row)) continue;
      if (!bw_kj_take(t, e.n_rec, 1, e.max_rows, BW_JW_FULL_EMIT, rec)) continue;
      u32 rb[BW_JW_MAXSIDES] = {0, 0, 0, 0}, rn[BW_JW_MAXSIDES] = {0, 0, 0, 0};
      for (int x = 0; x < t.sides; ++x) {
        rb[x] = c.gen[x];
        rn[x] = c.cnt[x] - c.gen[x];
      }
      bw_kj_event(e, p, t.sides, t.keys[s], c, row, 0, rec);
      bw_kj_stage(t, e, p, s, rec, rb, rn);
    }
    for (int x = 0; x < BW_JW_MAXSIDES; ++x) c.gen[x] = c.cnt[x];
    t.cell[s] = c;
  }
}

// after the per-key kernel of a call, over the whole store: an entry inside its key's stage record of this call is
// copied to staging; an entry whose rank its side's gen passed (EOF: every entry) dies and releases its handle.  Nothing
// to do when the call made no record and moved no gen (rec0: the records before the call), nor after a failed call
// (records may lack staging).
__global__ void k_kjoin_gather(KjTable t, KjEmit e, CwStore es, KjParams p, u64 rec0, unsigned long long* n_dead) {
  if (*t.err) return;
  if (!p.eof && *e.n_rec == rec0 && *e.n_kill == 0) return;
  const u64 n = *es.n;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  for (u64 b = (u64)blockIdx.x * blockDim.x; b < n; b += stride) {  // (b is warp-uniform: the whole warp reaches the ballots)
    const u64 i = b + threadIdx.x;
    bool dead = false;
    u64 h = 0;
    if (i < n) {
      const u64 r = es.ref[i];
      if (r != BW_CW_DEAD) {
        const u64 slot = r >> 2;
        const int s = (int)(r & 3);
        const u32 rank = es.rank[i];
        h = es.h[i];
        if (t.rec_ord[slot] == p.ord) {
          const u64 c = t.rec_c[slot];
          const u32 d = rank - e.rb[c * 4 + s];  // (wraps above every count when rank < b)
          if (d < e.rn[c * 4 + s]) e.stage[e.rbase[c * 4 + s] + d] = h;
        }
        if (p.eof || rank < t.cell[slot].gen[s]) {
          dead = true;
          es.ref[i] = BW_CW_DEAD;
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

__global__ void k_kjoin_init(KjTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.keys[s] = BW_EMPTY_KEY;
    t.cell[s] = KjCell{};
    t.live[s] = 0;
    t.rec_ord[s] = ~0ULL;
  }
}
