// bw_keyed.cuh -- K5 / K6: order-preserving per-key steps that are not window folds.
//
// K5 `bw_smap`: `stateful_map` with the rolling z-score detector of
//   examples/anomaly_detector.py:16-48 (BASELINE config C2).  The reference runs
//   `_StatefulLogic.on_batch` -> `_StatefulFlatMapLogic.on_item`
//   (operators/__init__.py:1024-1042, 2860-2890): one Python call per item, in
//   arrival order per key.  Here: stable sort of the activation by key (CUB),
//   then every item is independent -- its statistics depend only on the previous
//   N-1 values of the same key, which are its neighbours in the sorted order (or
//   the key's carried ring for the first N-1 items of a segment).
// K6 `bw_join`: two-sided keyed join, `_JoinLogic.on_item`
//   (operators/__init__.py:2157-2190) in insert modes first/last and emit modes
//   complete/running/final (BASELINE config C4).  Same grouping; one thread walks
//   a key's items of the activation in arrival order (segments are short: a join
//   key sees a handful of items).
#pragma once
#include "bw_common.cuh"

#define BW_SMAP_MAXW 32

struct SmapTable {
  u64* keys;     // BW_EMPTY_KEY when free; slot `cap` is the alias slot of that key value
  u32* cnt;      // values held in the ring (<= window)
  double* ring;  // [slot][window], newest first
  u64 cap;
  int window;
  u32* err;
};

__device__ __forceinline__ u64 bw_keyed_find(u64* keys, u64 cap, u64 key, u32* err) {
  if (key == BW_EMPTY_KEY) return cap;
  u64 s = bw_slot_of_hash(bw_mix64(key), cap);
  for (u64 probe = 0; probe < cap; ++probe) {
    u64 k = keys[s];
    if (k == key) return s;
    if (k == BW_EMPTY_KEY) {
      u64 old = atomicCAS((unsigned long long*)&keys[s], (unsigned long long)BW_EMPTY_KEY, (unsigned long long)key);
      if (old == BW_EMPTY_KEY || old == key) return s;
    }
    if (++s >= cap) s = 0;
  }
  atomicCAS(err, 0u, 3u);
  return ~0ULL;
}

// headpos[p] = sorted position of the first item of p's key (after an inclusive max-scan)
__global__ void k_keyed_heads(const u64* ksorted, u32* headpos, u64 n) {
  for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (u64)gridDim.x * blockDim.x)
    headpos[p] = (p == 0 || ksorted[p] != ksorted[p - 1]) ? (u32)p : 0u;
}

// slot of every segment (written at the head position)
__global__ void k_smap_slots(SmapTable t, const u64* ksorted, const u32* headpos, u64* slot_at_head, u64 n) {
  for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (u64)gridDim.x * blockDim.x)
    if (headpos[p] == p) slot_at_head[p] = bw_keyed_find(t.keys, t.cap, ksorted[p], t.err);
}

__device__ __forceinline__ double bw_val_f64(const void* vals, int is_f32, u64 i) {
  return is_f32 ? (double)((const float*)vals)[i] : ((const double*)vals)[i];
}

// CPython >= 3.12 `sum()` of floats: Neumaier compensated summation (Python/bltinmodule.c); the kernel adds the
// same way, so its sums, and so mu, are bit-identical to the reference mapper's on CPython >= 3.12.
struct PySum {
  double s = 0.0, c = 0.0;
  __device__ __forceinline__ void add(double x) {
    const double t = __dadd_rn(s, x);
    if (fabs(s) >= fabs(x)) c = __dadd_rn(c, __dadd_rn(__dsub_rn(s, t), x));
    else c = __dadd_rn(c, __dadd_rn(__dsub_rn(x, t), s));
    s = t;
  }
  __device__ __forceinline__ double result() const { return (c != 0.0 && isfinite(c)) ? __dadd_rn(s, c) : s; }
};

// mean / population sigma of `len` values produced by get(0..len-1), newest first
// (the order Python's sum() walks `last_10`); explicit round-to-nearest ops, no FMA contraction.
// mu is bit-identical to CPython >= 3.12.  The square and the sqrt are correctly rounded; the reference's `** 2` and
// `** 0.5` go through libm `pow`, which is not always, so sigma can differ from it by 1 ulp and a flag can differ
// only where z is within a few ulp of the threshold.  `po.run_zscore(..., correctly_rounded=True)` is the exact twin.
template <class Get>
__device__ __forceinline__ void bw_window_stats(Get get, int len, double& mu, double& sigma) {
  PySum a;
  for (int k = 0; k < len; ++k) a.add(get(k));
  mu = __ddiv_rn(a.result(), (double)len);
  PySum q;
  for (int k = 0; k < len; ++k) {
    const double d = __dsub_rn(get(k), mu);
    q.add(__dmul_rn(d, d));
  }
  sigma = __dsqrt_rn(__ddiv_rn(q.result(), (double)len));
}

__global__ void k_smap_eval(SmapTable t, const u32* isorted, const u32* headpos, const u64* slot_at_head, const void* vals,
                            int is_f32, double threshold, double* out_mu, double* out_sigma, unsigned char* out_flag, u64 n) {
  const int W = t.window;
  for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (u64)gridDim.x * blockDim.x) {
    const u64 h = headpos[p];
    const u64 s = slot_at_head[h];
    if (s == ~0ULL) continue;
    const int j = (int)(p - h);  // earlier items of this key inside this activation
    const int n0 = (int)t.cnt[s];
    const double* ring = t.ring + s * (u64)W;
    // value k steps back from position q (k = 0 is the item at q itself)
    auto back = [&](u64 q, int jq, int k) -> double {
      return (k <= jq) ? bw_val_f64(vals, is_f32, isorted[q - k]) : ring[k - jq - 1];
    };
    const double v = bw_val_f64(vals, is_f32, isorted[p]);
    // statistics BEFORE the push decide the flag (anomaly_detector.py:33-46)
    bool flag = false;
    int plen = j + n0;
    if (plen > W) plen = W;
    if (plen > 0) {
      double pm, ps;
      bw_window_stats([&](int k) { return back(p - 1, j - 1, k); }, plen, pm, ps);  // j == 0: every term comes from the ring
      if (pm != 0.0 && ps != 0.0) flag = __ddiv_rn(fabs(__dsub_rn(v, pm)), ps) > threshold;      // `if self.mu and self.sigma`
    }
    int len = j + 1 + n0;
    if (len > W) len = W;
    double mu, sigma;
    bw_window_stats([&](int k) { return back(p, j, k); }, len, mu, sigma);
    const u32 o = isorted[p];
    out_mu[o] = mu;
    out_sigma[o] = sigma;
    out_flag[o] = flag ? 1 : 0;
  }
}

// after the evaluation: the last item of every segment rewrites the key's ring
__global__ void k_smap_update(SmapTable t, const u64* ksorted, const u32* isorted, const u32* headpos, const u64* slot_at_head,
                              const void* vals, int is_f32, u64 n) {
  const int W = t.window;
  for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (u64)gridDim.x * blockDim.x) {
    if (p + 1 < n && ksorted[p + 1] == ksorted[p]) continue;  // not the tail
    const u64 h = headpos[p];
    const u64 s = slot_at_head[h];
    if (s == ~0ULL) continue;
    const int j = (int)(p - h);
    const int n0 = (int)t.cnt[s];
    double* ring = t.ring + s * (u64)W;
    double fresh[BW_SMAP_MAXW];
    int len = j + 1 + n0;
    if (len > W) len = W;
    for (int k = 0; k < len; ++k) fresh[k] = (k <= j) ? bw_val_f64(vals, is_f32, isorted[p - k]) : ring[k - j - 1];
    for (int k = 0; k < len; ++k) ring[k] = fresh[k];
    t.cnt[s] = (u32)len;
  }
}

// ---------------------------------------------------------------------------
// join
// ---------------------------------------------------------------------------
struct __align__(32) JoinSlot {
  u64 key;
  u64 l, r;
  u64 flags;  // bit0: left set, bit1: right set
};
struct JoinEmit {
  u64 *key, *l, *r, *mask, *seq, *epoch;
  u64 max_rows;
  unsigned long long* n_rows;
};
enum { BW_JOIN_FIRST = 0, BW_JOIN_LAST = 1 };
enum { BW_JOIN_COMPLETE = 0, BW_JOIN_FINAL = 1, BW_JOIN_RUNNING = 2 };

__device__ __forceinline__ u64 bw_join_find(JoinSlot* slots, u64 cap, u64 key, u32* err) {
  if (key == BW_EMPTY_KEY) return cap;
  u64 s = bw_slot_of_hash(bw_mix64(key), cap);
  for (u64 probe = 0; probe < cap; ++probe) {
    u64 k = slots[s].key;
    if (k == key) return s;
    if (k == BW_EMPTY_KEY) {
      u64 old = atomicCAS((unsigned long long*)&slots[s].key, (unsigned long long)BW_EMPTY_KEY, (unsigned long long)key);
      if (old == BW_EMPTY_KEY || old == key) return s;
    }
    if (++s >= cap) s = 0;
  }
  atomicCAS(err, 0u, 3u);
  return ~0ULL;
}

__device__ __forceinline__ void bw_join_emit(const JoinEmit& e, u32* err, u64 key, u64 l, u64 r, u64 mask, u64 seq, u64 epoch) {
  u64 i = atomicAdd(e.n_rows, 1ULL);
  if (i >= e.max_rows) {
    atomicCAS(err, 0u, 3u);
    return;
  }
  e.key[i] = key;
  e.l[i] = l;
  e.r[i] = r;
  e.mask[i] = mask;
  e.seq[i] = seq;
  e.epoch[i] = epoch;
}

// one thread per key segment: the key's items of this activation in arrival order
__global__ void k_join_apply(JoinSlot* slots, u64 cap, u32* err, const u64* ksorted, const u32* isorted, const u32* headpos,
                             const unsigned char* side, const u64* vals, u64 n, int insert_mode, int emit_mode, JoinEmit e,
                             u32 batch_no, u64 epoch) {
  for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (u64)gridDim.x * blockDim.x) {
    if (headpos[p] != p) continue;
    const u64 key = ksorted[p];
    const u64 s = bw_join_find(slots, cap, key, err);
    if (s == ~0ULL) continue;
    u64 l = slots[s].l, r = slots[s].r, fl = slots[s].flags;
    for (u64 q = p; q < n && ksorted[q] == key; ++q) {
      const u32 o = isorted[q];
      const int sd = side[o] ? 1 : 0;
      const u64 v = vals[o];
      const u64 bit = 1ULL << sd;
      if (insert_mode == BW_JOIN_LAST || !(fl & bit)) {
        if (sd) r = v; else l = v;
        fl |= bit;
      }
      const u64 seq = ((u64)batch_no << 32) | o;
      if (emit_mode == BW_JOIN_COMPLETE && fl == 3ULL) {
        bw_join_emit(e, err, key, l, r, 3ULL, seq, epoch);
        fl = 0;  // DISCARD: a later item starts from a fresh state
      } else if (emit_mode == BW_JOIN_RUNNING) {
        bw_join_emit(e, err, key, l, r, fl, seq, epoch);
      }
    }
    slots[s].l = l;
    slots[s].r = r;
    slots[s].flags = fl;
  }
}

__global__ void k_join_eof(JoinSlot* slots, u64 cap, u32* err, int emit_mode, JoinEmit e, u64 epoch) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= cap; s += (u64)gridDim.x * blockDim.x) {
    const u64 fl = slots[s].flags;
    if (!fl) continue;
    if (emit_mode == BW_JOIN_FINAL) bw_join_emit(e, err, s == cap ? BW_EMPTY_KEY : slots[s].key, slots[s].l, slots[s].r, fl, 0, epoch);
    slots[s].flags = 0;
  }
}

__global__ void k_join_init(JoinSlot* slots, u64 cap) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= cap; s += (u64)gridDim.x * blockDim.x) {
    JoinSlot j;
    j.key = BW_EMPTY_KEY;
    j.l = j.r = j.flags = 0;
    slots[s] = j;
  }
}
__global__ void k_smap_init(SmapTable t) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    t.keys[s] = BW_EMPTY_KEY;
    t.cnt[s] = 0;
  }
}
