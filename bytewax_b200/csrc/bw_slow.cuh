// bw_slow.cuh -- exact path for an activation that may contain late items, and
// the reference-order sort of emitted rows.
//
// Late detection restates windowing.py:1120-1130: item i of a key is late iff
//     ts_i < max(UTC_MIN, max(B_key, max_{j<i, same key} ts_j) - wait)
// where B_key is the key's running maximum before this activation.  The
// per-key prefix maximum in arrival order is a stable sort by key followed by
// an exclusive max-scan-by-key (CUB; this path is off the steady state).
// Late items are emitted once per window of `late_for(ts)`
// (windowing.py:636-637) and never folded; the rest goes through the same
// `bw_fold_event` as the fast path.
#pragma once
#include "bw_close.cuh"
#include "bw_common.cuh"
#include "bw_fold.cuh"
#include "bw_prepass.cuh"

// flatten segments: keys_flat[g], ts_flat[g], idx[g] = g
__global__ void k_slow_flatten(BatchView bv, FoldParams p, u64* keys_flat, i64* ts_flat, u32* idx) {
  __shared__ u64 seg_start[BW_MAX_WORLD + 1];
  if (threadIdx.x == 0) {
    u64 acc = 0;
    for (int j = 0; j < bv.nseg; ++j) {
      seg_start[j] = acc;
      acc += bw_seg_count(bv, j);
    }
    seg_start[bv.nseg] = acc;
  }
  __syncthreads();
  const u64 total = seg_start[bv.nseg];
  for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (u64)gridDim.x * blockDim.x) {
    int seg = 0;
    u64 off = g;
    if (bv.nseg > 1) bw_locate(bv, seg_start, g, seg, off);
    keys_flat[g] = bv.keys[seg][off];
    ts_flat[g] = bw_load_ts(bv, seg, off, p);
    idx[g] = (u32)g;
  }
}

__global__ void k_gather_i64(const i64* src, const u32* idx, i64* dst, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
    dst[i] = src[idx[i]];
}

// read-only lookup of a key's running max ts (INT64_MIN when the key has no state)
__device__ __forceinline__ i64 bw_lookup_max_ts(const Table& t, u64 key) {
  u64 s = bw_home_slot(t, key);
  if (key == BW_EMPTY_KEY) return t.hot[s].max_ts;
  for (u64 probe = 0; probe <= (u64)t.seg_mask; ++probe) {
    u64 k = t.hot[s].key;
    if (k == key) return t.hot[s].max_ts;
    if (k == BW_EMPTY_KEY) return INT64_MIN;
    s = bw_probe_next(t, s, 1);
  }
  return INT64_MIN;
}

// A key whose only items of an activation were late still had `on_batch` run (windowing.py:1115-1133): under a moving
// system clock its watermark may have grown since its last activation, so K4 has to look at it.
__device__ __forceinline__ void bw_wake_key(const Table& t, u64 key) {
  u64 s = bw_home_slot(t, key);
  if (key != BW_EMPTY_KEY) {
    u64 probe = 0;
    for (; probe <= (u64)t.seg_mask; ++probe) {
      const u64 k = t.hot[s].key;
      if (k == key) break;
      if (k == BW_EMPTY_KEY) return;
      s = bw_probe_next(t, s, 1);
    }
    if (probe > (u64)t.seg_mask) return;
  }
  if (t.hot[s].wt0 == BW_EMPTY_WIDTAG) return;  // no open window
  const unsigned long long old = atomicOr((unsigned long long*)&t.hot[s].wt0, (unsigned long long)BW_TAG_DIRTY);
  if (!(old & (unsigned long long)BW_TAG_DIRTY)) t.dirty[atomicAdd(&t.ctr->dirty_count, 1u)] = (u32)s;
}

// sorted order i -> late flag at arrival index
__global__ void k_slow_classify(Table t, FoldParams p, const u64* keys_sorted, const u32* idx_sorted,
                                const i64* ts_sorted, const i64* prefmax, unsigned char* late, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    i64 m = bw_lookup_max_ts(t, keys_sorted[i]);
    if (prefmax[i] > m) m = prefmax[i];
    const i64 wm = bw_wm_floor(bw_sub_sat(m, p.wait_us), p);  // (m == INT64_MIN: the floor)
    late[idx_sorted[i]] = (ts_sorted[i] < wm) ? 1 : 0;
  }
}

__global__ void __launch_bounds__(BW_FOLD_THREADS)
k_slow_fold(BatchView bv, Table t, FoldParams p, EmitBufs e, const unsigned char* late, u32 batch_no, u64 epoch) {
  __shared__ u64 seg_start[BW_MAX_WORLD + 1];
  __shared__ BlockSinks sinks;
  bw_sinks_init(&sinks);
  if (threadIdx.x == 0) {
    u64 acc = 0;
    for (int j = 0; j < bv.nseg; ++j) {
      seg_start[j] = acc;
      acc += bw_seg_count(bv, j);
    }
    seg_start[bv.nseg] = acc;
  }
  __syncthreads();
  const u64 total = seg_start[bv.nseg];
  for (u64 base = (u64)blockIdx.x * blockDim.x; base < total; base += (u64)gridDim.x * blockDim.x) {
    u64 g = base + threadIdx.x;
    if (g < total) {
      int seg = 0;
      u64 off = g;
      if (bv.nseg > 1) bw_locate(bv, seg_start, g, seg, off);
      u64 key, operand, raw;
      i64 ts;
      bw_load_event(bv, seg, off, p, key, ts, operand, raw);
      const u64 seq = ((u64)batch_no << 32) | g;
      if (!late[g]) {
        bw_fold_event<FoldCfgRuntime>(t, p, &sinks, key, ts, operand, seq, batch_no, BW_NO_SLOT);
      } else {
        // late_for(ts) == intersects(ts): floor((d-length)/offset)+1 .. floor(d/offset)
        i64 d = ts - p.align_us;
        i64 w0 = bw_floordiv(d - p.length_us, p.offset_us) + 1;
        i64 w1 = bw_floordiv(d, p.offset_us);
        u32 nw = (w1 >= w0) ? (u32)(w1 - w0 + 1) : 0u;
        if (p.now_us != 0) bw_wake_key(t, key);
        u64 at = bw_warp_reserve(&t.ctr->n_late, nw);
        if (at + nw > e.max_late) {
          bw_raise(t.ctr, 3u);
        } else {
          // late rows carry the raw value bits widened to 64 (f32 -> f64 bits)
          u64 vbits = raw;
          if (p.val_dtype == 2) vbits = (u64)__double_as_longlong((double)__uint_as_float((u32)raw));
          for (u32 j = 0; j < nw; ++j) {
            e.l_key[at + j] = key;
            e.l_wid[at + j] = w0 + j;
            e.l_val[at + j] = vbits;
            e.l_ts[at + j] = ts + p.now_us;  // (back from the frame where system time is 0)
            e.l_seq[at + j] = seq;
            e.l_epoch[at + j] = epoch;
          }
        }
      }
    }
    __syncthreads();
    if (sinks.n_dirty > BW_SINK_CAP / 2) bw_sinks_flush(&sinks, t);
  }
  __syncthreads();
  bw_sinks_flush(&sinks, t);
}

// ---------------------------------------------------------------------------
// Reference emission order: ascending key *string* (decimal text of the u64),
// then first-opened order.  Decimal-text order of u64 == order of
// (first 19 digits left-aligned, digit count, 20th digit).
// ---------------------------------------------------------------------------
__constant__ u64 BW_P10[20] = {1ULL,
                               10ULL,
                               100ULL,
                               1000ULL,
                               10000ULL,
                               100000ULL,
                               1000000ULL,
                               10000000ULL,
                               100000000ULL,
                               1000000000ULL,
                               10000000000ULL,
                               100000000000ULL,
                               1000000000000ULL,
                               10000000000000ULL,
                               100000000000000ULL,
                               1000000000000000ULL,
                               10000000000000000ULL,
                               100000000000000000ULL,
                               1000000000000000000ULL,
                               10000000000000000000ULL};

__device__ __forceinline__ int bw_ndigits(u64 k) {
  int d = 1;
#pragma unroll
  for (int i = 1; i < 20; ++i)
    if (k >= BW_P10[i]) d = i + 1;
  return d;
}

enum { BW_SK_SEQ = 0, BW_SK_DIGITS = 1, BW_SK_ALIGNED = 2, BW_SK_EPOCH = 3, BW_SK_WID = 4 };

__global__ void k_sortkey(int kind, const u64* key, const u64* seq, const u64* epoch, const i64* wid,
                          const u32* perm, u64* out, u64 n, u64 epoch_base) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    u32 r = perm[i];
    u64 v;
    if (kind == BW_SK_SEQ) {
      v = seq[r];
    } else if (kind == BW_SK_EPOCH) {
      v = epoch[r] - epoch_base;
    } else if (kind == BW_SK_WID) {
      v = (u64)wid[r] ^ 0x8000000000000000ULL;
    } else {
      u64 k = key[r];
      int d = bw_ndigits(k);
      if (kind == BW_SK_DIGITS)
        v = ((u64)d << 4) | (d == 20 ? (k % 10ULL) : 0ULL);
      else
        v = (d == 20) ? (k / 10ULL) : k * BW_P10[19 - d];
    }
    out[i] = v;
  }
}

__global__ void k_iota(u32* p, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) p[i] = (u32)i;
}
__global__ void k_gather_u64(const u64* src, const u32* perm, u64* dst, u64 n) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
    dst[i] = src[perm[i]];
}
