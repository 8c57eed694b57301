// bw_kcollect.cuh -- K13: the window-free keyed `collect(step_id, up, timeout, max_size)`.
//
// The reference runs `_CollectLogic` (pysrc/bytewax/operators/__init__.py:1113-1164) under `stateful` (:1025-1062):
// per key a list `acc` and a `timeout_at`; every item sets timeout_at = now + timeout and appends; a list that reaches
// max_size is emitted and the logic discarded, so the key's next item, even in the same batch, starts a fresh list.  A
// notify (src/operators.rs:808-858) or EOF (:862-894) emits the list and discards the key.
//
// Where a key's lists split depends only on each value's position in the key's sequence, so no thread walks a key.
// With c0 the key's carried count and M = max_size, row i of the key's segment of a call has position p = c0 + i; list
// j = p / M is complete when (j + 1) * M <= c0 + n.  One thread per segment (at its tail, which knows the segment's
// length) reserves the key's complete lists -- records and a staging range, by atomics -- and the carry's new entries;
// then every row goes to its place on its own (k_kcol_rows): the staging range at `base + p`, or the key's carry.
// Carried handles only ever fill list 0; they move from the carry to `base + rank` in k_kcol_gather, over the whole
// entry store, so a 10^6-item key is placed by the whole grid either way.
//
// The carry is K9's entry store (bw_collect.cuh: CwStore, with its growth and compaction, host side): one entry per
// carried value, ref = the key's slot, rank = the value's position in the key's list.  The staging buffer and its CSR
// placement at advance / eof are K9's too (records, k_cwin_order, k_cwin_place).
#pragma once
#include "../../include/bwgpu.h"
#include "bw_collect.cuh"
#include "bw_keyed.cuh"

struct KcTable {
  u64* keys;     // BW_EMPTY_KEY when free; slot `cap` is the alias slot of that key value
  u64* cnt;      // carried handles (0: no live logic)
  i64* due;      // timeout_at of the carry (meaningless while cnt == 0)
  u64* mv_ord;   // the call in which the carry last moved to a list
  u64* mv_base;  // ... and its staging position and record
  u64* mv_rec;
  u64 cap;
  u64 M;         // max_size >= 1
  // the fail helper of bw_jwin.cuh reads these two
  u32* err;
  u32* why;
};
struct KcEmit {  // complete or timed-out lists: one record each; its handles at stage[soff, soff + cnt)
  u64 *key, *cnt, *soff, *epoch, *ord, *seq;
  u64 max_rows;
  unsigned long long* n_rows;
  u64* stage;
  u32* stage_rec;
  u64 max_stage;
  unsigned long long* n_stage;
  unsigned long long* n_moved;  // carried entries moved out in this call (the gather runs only when some did)
};
struct KcSeg {  // one key segment of a call, at its head position
  u64 slot;     // ~0: the key found no slot or its lists no room; its rows are dropped and the call fails
  u64 c0;       // carried before the call
  u64 cut;      // handles in complete lists
  u64 base;     // staging position of the first complete list
  u64 rec;      // record of the first complete list
  u64 sbase;    // store index of the first new carry entry
};
struct KcParams {
  u64 epoch, ord;
  i64 timeout_at;
};

__device__ __forceinline__ void bw_kc_record(const KcEmit& e, const KcParams& p, u64 c, u64 key, u64 cnt, u64 soff, u64 seq) {
  e.key[c] = key;
  e.cnt[c] = cnt;
  e.soff[c] = soff;
  e.epoch[c] = p.epoch;
  e.ord[c] = p.ord;
  e.seq[c] = seq;
}

// a key's carried handles go to list 0 of this call at `base`, record `rec`
__device__ __forceinline__ void bw_kc_move(const KcTable& t, const KcEmit& e, const KcParams& p, u64 s, u64 c0, u64 base, u64 rec) {
  t.mv_ord[s] = p.ord;
  t.mv_base[s] = base;
  t.mv_rec[s] = rec;
  atomicAdd(e.n_moved, (unsigned long long)c0);
}

// one thread per key segment, at its tail: the key's slot, complete lists, new carry and timeout
__global__ void k_kcol_keys(KcTable t, KcEmit e, CwStore es, KcParams p, KcSeg* seg, const u64* ksorted, const u32* headpos, u64 n) {
  for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (u64)gridDim.x * blockDim.x) {
    if (q + 1 < n && ksorted[q + 1] == ksorted[q]) continue;  // not the tail
    const u64 h = headpos[q];
    KcSeg g{~0ULL, 0, 0, 0, 0, 0};
    const u64 s = bw_keyed_find(t.keys, t.cap, ksorted[q], t.err);
    if (s == ~0ULL) {
      bw_jw_fail(t, BW_JW_FULL_TABLE);
      seg[h] = g;
      continue;
    }
    const u64 c0 = t.cnt[s], total = c0 + (q - h + 1);
    const u64 lists = total / t.M;
    g.c0 = c0;
    g.cut = lists * t.M;
    const u64 carry = total - g.cut;
    const u64 adds = carry - (lists ? 0 : c0);  // new rows that join the carry
    if (carry >> 32) {  // (a rank is 32 bits: ~4.3e9 carried values, more than the store can hold on one GPU)
      bw_jw_fail(t, BW_CW_FULL_STORE);
      seg[h] = g;
      continue;
    }
    if (lists) {
      g.rec = atomicAdd(e.n_rows, (unsigned long long)lists);
      if (g.rec + lists > e.max_rows) {
        bw_jw_fail(t, BW_JW_FULL_EMIT);
        seg[h] = g;
        continue;
      }
      g.base = atomicAdd(e.n_stage, (unsigned long long)g.cut);
      if (g.base + g.cut > e.max_stage) {  // (sized by the host for every handle a call can stage: never reached)
        bw_jw_fail(t, BW_CW_FULL_STORE);
        seg[h] = g;
        continue;
      }
      if (c0) bw_kc_move(t, e, p, s, c0, g.base, g.rec);
    }
    g.sbase = adds ? atomicAdd(es.n, (unsigned long long)adds) : 0;
    if (g.sbase + adds > es.cap) {  // (sized by the host for every row of a call: never reached)
      bw_jw_fail(t, BW_CW_FULL_STORE);
      seg[h] = g;
      continue;
    }
    g.slot = s;
    seg[h] = g;
    t.cnt[s] = carry;
    if (carry) t.due[s] = p.timeout_at;
  }
}

// one thread per row: into its complete list's staging slot (the list's last row writes its record), or into the carry
__global__ void k_kcol_rows(KcTable t, KcEmit e, CwStore es, KcParams p, const KcSeg* seg, const u64* ksorted, const u32* isorted,
                            const u32* headpos, const u64* handles, u64 n) {
  for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (u64)gridDim.x * blockDim.x) {
    const u64 h = headpos[q];
    const KcSeg g = seg[h];
    if (g.slot == ~0ULL) continue;
    const u64 pos = g.c0 + (q - h);
    const u64 hd = handles[isorted[q]];
    if (pos < g.cut) {
      const u64 j = pos / t.M;
      e.stage[g.base + pos] = hd;
      e.stage_rec[g.base + pos] = (u32)(g.rec + j);
      if (pos + 1 == (j + 1) * t.M) bw_kc_record(e, p, g.rec + j, ksorted[q], t.M, g.base + j * t.M, j);
    } else {
      const u64 i = g.sbase + (pos - (g.cut > g.c0 ? g.cut : g.c0));
      es.ref[i] = g.slot;
      es.rank[i] = (u32)(pos - g.cut);
      es.h[i] = hd;
    }
  }
}

// advance / eof, one thread per slot: a key whose carry is due (eof: every live key) emits it as one list and resets
__global__ void k_kcol_due(KcTable t, KcEmit e, KcParams p, i64 now, int eof) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    const u64 c = t.cnt[s];
    if (!c || (!eof && t.due[s] > now)) continue;
    const u64 r = atomicAdd(e.n_rows, 1ULL);
    if (r >= e.max_rows) {
      bw_jw_fail(t, BW_JW_FULL_EMIT);
      continue;
    }
    const u64 at = atomicAdd(e.n_stage, (unsigned long long)c);
    if (at + c > e.max_stage) {  // (sized by the host for every carried handle: never reached)
      bw_jw_fail(t, BW_CW_FULL_STORE);
      continue;
    }
    bw_kc_record(e, p, r, t.keys[s], c, at, 0);
    bw_kc_move(t, e, p, s, c, at, r);
    t.cnt[s] = 0;
  }
}

// every carried entry of a key whose carry moved in this call goes to its list's staging slot and is dead
__global__ void k_kcol_gather(KcTable t, KcEmit e, CwStore es, KcParams p, u64 n) {
  if (*e.n_moved == 0) return;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const u64 s = es.ref[i];
    if (s == BW_CW_DEAD || t.mv_ord[s] != p.ord) continue;
    const u64 j = t.mv_base[s] + es.rank[i];
    e.stage[j] = es.h[i];
    e.stage_rec[j] = (u32)t.mv_rec[s];
    es.ref[i] = BW_CW_DEAD;
  }
}

__global__ void k_kcol_init(KcTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.keys[s] = BW_EMPTY_KEY;
    t.cnt[s] = 0;
    t.mv_ord[s] = ~0ULL;
  }
}
