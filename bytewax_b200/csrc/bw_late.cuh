// bw_late.cuh -- an activation with a few late rows, without sorting it.
//
// Row i of key k is late iff  ts_i < wm(max(B_k, P_i)),  B_k the key's running maximum before the activation and
// P_i the largest timestamp among the key's EARLIER rows of the activation (windowing.py:1120-1130, clock
// windowing.py:263-287; wm(m) = max(UTC_MIN, m - wait), UTC_MIN in absolute time: bw_wm_floor).  The exact path of
// bw_slow.cuh gets every P_i from a stable sort by key over the whole activation.  But only a SUSPECT row -- one behind the running maximum G_i over
// all keys, ts_i < wm(G_i), which is what made the verdict "not clean" -- can be late at all (P_i, B_k <= G_i), and
// an in-order stream with stragglers has few of them.  So:
//
//   k_late_gpre      exclusive running maximum at every tile start, from the tile maxima the scatter already has
//   k_late_suspect   per row, exact G_i (prefix maximum in arrival order: tile starts, the scatter's 64-row chunk maxima,
//                    a warp scan inside the chunk); suspects go into a small hash table keyed by key (duplicates
//                    allowed, generation-stamped: never cleared) and set a bit in a key filter
//   k_late_build     the suspects into the table, one thread each
//   k_late_prefmax   one pass over the keys: a row whose key passes the filter raises P of every suspect of that key
//                    that arrives after it (a hashed semi-join instead of a sort)
//   k_late_classify  suspect by suspect: late or not; late rows set their bit in a row bitmap
//   (host)           the scatter runs again, skipping the rows of the bitmap: what is left has no late row, so the
//                    streaming fold is exact for it -- late rows never raise a maximum, so dropping them changes no
//                    other row's verdict
//   k_late_emit      late rows out, one per window of late_for(ts) (windowing.py:636-637)
//
// Too many suspects for the table (heavily disordered input): the host takes the sort path instead.
#pragma once
#include "bw_close.cuh"
#include "bw_common.cuh"
#include "bw_fold.cuh"
#include "bw_prepass.cuh"
#include "bw_slow.cuh"

#define BW_LATE_TILE 2048  // == BW_SC_TILE: the scatter's lateness triples are per tile of this many rows ...
#define BW_LATE_CHUNK 64   // ... and it also leaves the maximum of every 64-row chunk (one per scatter warp): 32 per tile
#define BW_LATE_PROBE_MAX 4096u  // (a key with this many suspect rows in one activation: the sort path)

// one suspect row: a 32-byte sector
struct __align__(32) LateEnt {
  u64 key;
  i64 ts;
  i64 pmax;   // largest timestamp among the key's earlier rows of the activation
  u32 idx;    // arrival index
  u32 stamp;  // generation << 2 | state (1 suspect, 2 late); another generation: free (no clearing between activations)
};

struct LateBufs {
  u32* key_bits;   // filter over keys with a suspect row: bit (mix64(key) >> 32) & kb_mask
  u32 kb_mask;
  u32* late_bits;  // one bit per row of the activation
  LateEnt* ent;    // suspects, open addressing on mix64(key) & m_mask, one entry per suspect ROW
  u32 m_mask;
  u32 cap;         // suspects the table takes (load <= 1/2)
  u32 gen;         // this activation's generation (> 0)
  u32* counters;   // [0] suspects seen, [1] an insertion gave up (table full)
  // the suspects as k_late_suspect finds them (compact, any order); k_late_build puts them in the table
  u64* s_key;
  i64* s_ts;
  u32* s_idx;
  u32* s_slot;     // where k_late_build put it
  i64* gpre;       // per tile: running maximum over everything before the tile
};

__device__ __forceinline__ i64 bw_wm_of(i64 m, const FoldParams& p) {
  return bw_wm_floor(bw_sub_sat(m, p.wait_us), p);  // (m == INT64_MIN: the floor)
}

// one block: gpre[t] = max(gprev, tile_max[0..t))
__global__ void __launch_bounds__(1024) k_late_gpre(const i64* tile_max, u32 ntiles, i64 gprev, i64* gpre) {
  __shared__ i64 s_w[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const u32 per = (ntiles + 1023u) / 1024u;
  const u32 lo = min(threadIdx.x * per, ntiles), hi = min(lo + per, ntiles);
  i64 m = INT64_MIN;
  for (u32 t = lo; t < hi; ++t) m = max(m, tile_max[t]);
  i64 inc = m;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const i64 y = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc = max(inc, y);
  }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  i64 run = gprev;
  for (int w = 0; w < warp; ++w) run = max(run, s_w[w]);
  const i64 prev = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane > 0) run = max(run, prev);
  for (u32 t = lo; t < hi; ++t) {
    gpre[t] = run;
    run = max(run, tile_max[t]);
  }
}

// one warp per tile: chunk_pre[t][w] = max(gpre[t], chunk_max[t][0..w)) -- the running maximum before every 64-row chunk
__global__ void __launch_bounds__(256) k_late_chunkpre(const i64* chunk_max, const i64* gpre, u32 ntiles, i64* chunk_pre) {
  const int lane = threadIdx.x & 31;
  const u32 gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (u32 t = gw; t < ntiles; t += nw) {
    i64 inc = chunk_max[(u64)t * 32 + lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const i64 y = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc = max(inc, y);
    }
    const i64 prev = __shfl_up_sync(0xffffffffu, inc, 1);
    const i64 g0 = gpre[t];
    chunk_pre[(u64)t * 32 + lane] = (lane > 0) ? max(g0, prev) : g0;
  }
}

__device__ __forceinline__ u32 bw_late_insert(const LateBufs& L, u64 key, u32 idx, i64 ts) {
  const u64 mx = bw_mix64(key);
  const u32 bit = (u32)(mx >> 32) & L.kb_mask;
  atomicOr(&L.key_bits[bit >> 5], 1u << (bit & 31u));
  u32 s = (u32)mx & L.m_mask;
  const u32 mine = (L.gen << 2) | 1u;
  for (u32 tries = 0; tries < BW_LATE_PROBE_MAX; ++tries) {
    u32 st = L.ent[s].stamp;
    bool got = false;
    while ((st >> 2) != L.gen) {  // free (an older generation): claim it
      const u32 old = atomicCAS(&L.ent[s].stamp, st, mine);
      if (old == st) {
        got = true;
        break;
      }
      st = old;
    }
    if (got) {
      L.ent[s].key = key;
      L.ent[s].ts = ts;
      L.ent[s].pmax = INT64_MIN;
      L.ent[s].idx = idx;
      return s;
    }
    s = (s + 1u) & L.m_mask;
  }
  L.counters[1] = 1u;  // (more suspects than the table was sized for: the host takes the sort path)
  return 0xFFFFFFFFu;
}

// A warp takes 64 consecutive rows at a time (two per lane: 128-bit loads), four such chunks in flight; no block
// barrier.  Exact running maximum before every row = what came before its chunk (chunk_pre) and the earlier lanes'
// pairs.  A chunk that is in order and starts at or after the watermark of what came before it has no suspect.
#define BW_LATE_SQ 128  // suspects a warp collects in shared memory before it reserves room in the list (one atomic on ONE
                        // word per reservation: they serialise in L2, ~2 ns each -- per warp and step that was the whole kernel)
__global__ void __launch_bounds__(256) k_late_suspect(BatchView bv, FoldParams p, u64 n, const i64* chunk_pre, LateBufs L) {
  __shared__ u64 qk[8][BW_LATE_SQ];
  __shared__ i64 qt[8][BW_LATE_SQ];
  __shared__ u32 qi[8][BW_LATE_SQ];
  const int warp = threadIdx.x >> 5;
  u32 qn = 0;  // (warp-uniform)
  auto flush = [&]() {
    if (qn == 0) return;
    __syncwarp();
    u32 base = 0;
    if ((threadIdx.x & 31) == 0) base = atomicAdd(&L.counters[0], qn);
    base = __shfl_sync(0xffffffffu, base, 0);
    for (u32 q = threadIdx.x & 31; q < qn; q += 32)
      if (base + q < L.cap) {  // (else: the host sees the count and takes the sort path)
        L.s_key[base + q] = qk[warp][q];
        L.s_ts[base + q] = qt[warp][q];
        L.s_idx[base + q] = qi[warp][q];
      }
    __syncwarp();
    qn = 0;
  };
  const int lane = threadIdx.x & 31;
  const u64 gw = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((u64)gridDim.x * blockDim.x) >> 5;
  const u64 ntask = (n + BW_LATE_CHUNK - 1) / BW_LATE_CHUNK;
  const u64* col = p.ts_from_value ? (const u64*)bv.vals[0] : (const u64*)bv.ts[0];
  const i64 add = p.ts_from_value ? p.align_us : -p.now_us;
  // (the next step's loads are issued before this step's rows are looked at: the memory system stays busy while the
  // warp scans)
  auto load4 = [&](u64 t0, i64* ta, i64* tb, i64* pre) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const u64 task = t0 + (u64)u * nw;
      const u64 r = task * BW_LATE_CHUNK + 2 * (u64)lane;
      ta[u] = INT64_MAX;  // (rows past the end: never suspect, never break the order)
      tb[u] = INT64_MAX;
      pre[u] = INT64_MIN;
      if (r + 1 < n) {
        u64 a, b;
        bw_ld_stream_2u64(col + r, a, b);
        ta[u] = add + (i64)a;
        tb[u] = add + (i64)b;
      } else if (r < n) {
        ta[u] = add + (i64)col[r];
      }
      if (task < ntask) pre[u] = chunk_pre[task];
    }
  };
  i64 na[4], nb[4], npre[4];
  if (gw < ntask) load4(gw, na, nb, npre);
  for (u64 t0 = gw; t0 < ntask; t0 += 4 * nw) {
    i64 ta[4], tb[4], pre[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      ta[u] = na[u];
      tb[u] = nb[u];
      pre[u] = npre[u];
    }
    if (t0 + 4 * nw < ntask) load4(t0 + 4 * nw, na, nb, npre);
    u32 sus = 0;  // bit 2u: row a of chunk u is a suspect, bit 2u + 1: row b
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const u64 task = t0 + (u64)u * nw;
      if (task >= ntask) break;
      const i64 wm0 = bw_wm_of(pre[u], p);
      const i64 nxt = __shfl_down_sync(0xffffffffu, ta[u], 1);
      const bool fine = ta[u] <= tb[u] && (lane == 31 || tb[u] <= nxt) && ta[u] >= wm0;
      if (__all_sync(0xffffffffu, fine)) continue;  // in order, and nothing behind what came before
      const u64 r = task * BW_LATE_CHUNK + 2 * (u64)lane;
      const i64 va = (r < n) ? ta[u] : INT64_MIN, vb = (r + 1 < n) ? tb[u] : INT64_MIN;
      i64 inc = max(va, vb);
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const i64 y = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc = max(inc, y);
      }
      const i64 prev = __shfl_up_sync(0xffffffffu, inc, 1);
      const i64 ga = (lane > 0) ? max(pre[u], prev) : pre[u];
      if (r < n && va < bw_wm_of(ga, p)) sus |= 1u << (2 * u);
      if (r + 1 < n && vb < bw_wm_of(max(ga, va), p)) sus |= 2u << (2 * u);
    }
    // the warp's suspects of these four chunks: into its queue (or, too many for it, straight to the list)
    if (__any_sync(0xffffffffu, sus != 0u)) {
      const u32 mine = (u32)__popc(sus);
      u32 incl = mine;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += y;
      }
      const u32 total = __shfl_sync(0xffffffffu, incl, 31);
      if (qn + total > BW_LATE_SQ) flush();
      const bool direct = total > BW_LATE_SQ;
      u32 base = 0;
      if (direct) {
        if (lane == 0) base = atomicAdd(&L.counters[0], total);
        base = __shfl_sync(0xffffffffu, base, 0);
      }
      u32 at = (direct ? base : qn) + incl - mine;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const u64 r = (t0 + (u64)u * nw) * BW_LATE_CHUNK + 2 * (u64)lane;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!(sus & ((1u << h) << (2 * u)))) continue;
          const u64 key = bv.keys[0][r + h];
          const i64 ts = h ? tb[u] : ta[u];
          if (!direct) {
            qk[warp][at] = key;
            qt[warp][at] = ts;
            qi[warp][at] = (u32)(r + h);
          } else if (at < L.cap) {
            L.s_key[at] = key;
            L.s_ts[at] = ts;
            L.s_idx[at] = (u32)(r + h);
          }
          ++at;
        }
      }
      if (!direct) qn += total;
    }
  }
  flush();
}

// one thread per suspect: into the table
__global__ void __launch_bounds__(256) k_late_build(LateBufs L) {
  const u32 ns = L.counters[0];
  if (ns > L.cap) return;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x)
    L.s_slot[i] = bw_late_insert(L, L.s_key[i], L.s_idx[i], L.s_ts[i]);
}

// Every row tells the suspects of its key that arrive after it how new it is.  The rows whose key passes the filter
// (one in six when 1 % of the rows are suspects) are queued per warp and handled by consecutive lanes: the probe loop
// runs once per 128 rows of the warp, not once per 32 with most lanes idle.
#define BW_LATE_Q 256
__global__ void __launch_bounds__(256) k_late_prefmax(BatchView bv, FoldParams p, u64 n, LateBufs L) {
  if (L.counters[0] > L.cap || L.counters[1]) return;
  __shared__ u64 q_key[8][BW_LATE_Q];
  __shared__ u32 q_idx[8][BW_LATE_Q];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const u32 lt = (1u << lane) - 1u;
  u64 nkey[8];
  auto load8 = [&](u64 i0, u64* key) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const u64 i = i0 + (u64)u * stride;
      key[u] = (i < n) ? bw_ld_stream_u64(bv.keys[0] + i) : 0ULL;
    }
  };
  load8((u64)blockIdx.x * blockDim.x + threadIdx.x, nkey);
  for (u64 i0 = (u64)blockIdx.x * blockDim.x + threadIdx.x; i0 - threadIdx.x < n; i0 += 8 * stride) {  // (warp-uniform trip count)
    u64 key[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) key[u] = nkey[u];
    load8(i0 + 8 * stride, nkey);  // (the next step's keys are on their way while this step probes)
    u32 word[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {  // the filter words of all eight, before any is looked at
      const u32 bit = (u32)(bw_mix64(key[u]) >> 32) & L.kb_mask;
      word[u] = L.key_bits[bit >> 5] >> (bit & 31u);
    }
    u32 cnt = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const u64 i = i0 + (u64)u * stride;
      const bool hit = i < n && (word[u] & 1u);
      const u32 m = __ballot_sync(0xffffffffu, hit);
      if (hit) {
        const u32 at = cnt + __popc(m & lt);
        q_key[warp][at] = key[u];
        q_idx[warp][at] = (u32)i;
      }
      cnt += __popc(m);
    }
    __syncwarp();
    for (u32 q = (u32)lane; q < cnt; q += 32) {
      const u64 k = q_key[warp][q];
      const u32 i = q_idx[warp][q];
      u32 s = (u32)bw_mix64(k) & L.m_mask;
      LateEnt x = L.ent[s];
      const i64 ts = bw_load_ts(bv, 0, i, p);
      while ((x.stamp >> 2) == L.gen) {
        if (x.key == k && x.idx > i) atomicMax((long long*)&L.ent[s].pmax, (long long)ts);
        s = (s + 1u) & L.m_mask;
        x = L.ent[s];
      }
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(256) k_late_classify(Table t, FoldParams p, LateBufs L) {
  const u32 ns = L.counters[0];
  if (ns > L.cap || L.counters[1]) return;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
    const u32 s = L.s_slot[i];
    const LateEnt x = L.ent[s];
    i64 m = bw_lookup_max_ts(t, x.key);
    if (x.pmax > m) m = x.pmax;
    if (x.ts < bw_wm_of(m, p)) {
      L.ent[s].stamp = (L.gen << 2) | 2u;
      atomicOr(&L.late_bits[x.idx >> 5], 1u << (x.idx & 31u));
    }
  }
}

// Late rows out: one per window of late_for(ts) == intersects(ts): floor((d-length)/offset)+1 .. floor(d/offset).
// 1024 suspects per block and step, one reservation in the late stream for all of them.
__global__ void __launch_bounds__(256) k_late_emit(BatchView bv, Table t, FoldParams p, EmitBufs e, LateBufs L, u32 batch_no, u64 epoch) {
  __shared__ u32 s_n;
  __shared__ unsigned long long s_base;
  const u32 ns = L.counters[0];
  for (u32 s0 = blockIdx.x * 1024u; s0 < ns; s0 += gridDim.x * 1024u) {  // (uniform trip count: barriers inside)
    LateEnt x[4];
    u32 nw[4], tot = 0;
    i64 w0[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const u32 i = s0 + (u32)u * 256u + threadIdx.x;
      nw[u] = 0;
      w0[u] = 0;
      x[u].stamp = 0u;
      if (i < ns) x[u] = L.ent[L.s_slot[i]];
      if (x[u].stamp == ((L.gen << 2) | 2u)) {
        const i64 d = x[u].ts - p.align_us;
        w0[u] = bw_floordiv(d - p.length_us, p.offset_us) + 1;
        const i64 w1 = bw_floordiv(d, p.offset_us);
        nw[u] = (w1 >= w0[u]) ? (u32)(w1 - w0[u] + 1) : 0u;
        tot += nw[u];
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0u;
    __syncthreads();
    u32 off = 0;
    if (tot) off = atomicAdd(&s_n, tot);
    __syncthreads();
    if (threadIdx.x == 0 && s_n) s_base = atomicAdd(&t.ctr->n_late, (unsigned long long)s_n);
    __syncthreads();
    if (!tot) continue;
    u64 at = s_base + off;
    if (at + tot > e.max_late) {
      bw_raise(t.ctr, 3u);
      continue;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (!nw[u]) continue;
      const u32 i = x[u].idx;
      if (p.now_us != 0) bw_wake_key(t, x[u].key);
      u64 raw = 0;
      if (bv.vals[0]) raw = (p.val_dtype == 2) ? (u64)((const u32*)bv.vals[0])[i] : ((const u64*)bv.vals[0])[i];
      // late rows carry the raw value bits widened to 64 (f32 -> f64 bits)
      u64 vbits = raw;
      if (p.val_dtype == 2) vbits = (u64)__double_as_longlong((double)__uint_as_float((u32)raw));
      const u64 seq = ((u64)batch_no << 32) | i;
      for (u32 j = 0; j < nw[u]; ++j) {
        e.l_key[at + j] = x[u].key;
        e.l_wid[at + j] = w0[u] + j;
        e.l_val[at + j] = vbits;
        e.l_ts[at + j] = x[u].ts + p.now_us;  // (back from the frame where system time is 0)
        e.l_seq[at + j] = seq;
        e.l_epoch[at + j] = epoch;
      }
      at += nw[u];
    }
  }
}
