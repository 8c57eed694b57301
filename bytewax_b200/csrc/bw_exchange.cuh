// bw_exchange.cuh -- K1/K2: key hash, radix partition by owning rank, exchange.
//
// Replaces `PartitionOp::partition` (src/timely.rs:494-569: hash % workers)
// and the Timely `Exchange` pact behind `routed_exchange`
// (src/timely.rs:809-815), whose inter-process leg pickles every item and
// ships it over TCP (src/pyo3_extensions.rs:85-105).
//
// Three kernels per activation on each rank:
//   k_part_hist     per-tile histogram of destinations (packed 16-bit counters)
//   k_part_scan     exclusive scan over tiles -> stable offsets; publishes the
//                   per-destination row counts (P2P: straight into the peer's
//                   count table)
//   k_part_scatter  stable scatter of the columns.  In P2P mode the stores go
//                   directly into the owning rank's receive region over NVLink
//                   (CUDA-IPC mapped peer pointers): partition and exchange are
//                   one pass, no send buffer, no host-visible counts.
// Arrival order at the destination is (source rank, source order), a legal
// order under the reference (Timely gives none across workers, SURVEY 8e).
#pragma once
#include "bw_common.cuh"

#define BW_PART_THREADS 256
#define BW_PART_PER_THREAD 8
#define BW_PART_TILE (BW_PART_THREADS * BW_PART_PER_THREAD)

struct PartIn {
  const u64* keys;
  const void* vals;  // may be NULL
  const i64* ts;     // may be NULL
  u64 n;
  int val_bytes;     // 0, 4 or 8
  int world;
};
struct PartOut {
  u64* keys[BW_MAX_WORLD];  // destination d's region for THIS source rank
  void* vals[BW_MAX_WORLD];
  i64* ts[BW_MAX_WORLD];
  u64* counts[BW_MAX_WORLD];  // where to publish "rows from this rank" at destination d
  u64 region_cap;
  u32* rows[BW_MAX_WORLD];    // k_part_scatter<true>: each row's index in this rank's columns
};
// k_part_scatter<true, true>: a one-byte column that travels with the rows (the side of a windowed join row, K8)
struct PartSide {
  const unsigned char* src;         // this rank's column
  unsigned char* dst[BW_MAX_WORLD];  // destination d's region for this source rank
};

__device__ __forceinline__ u32 bw_dest_of(u64 key, int world) { return bw_route_hash(bw_mix64(key), (u32)world); }

__global__ void __launch_bounds__(BW_PART_THREADS) k_part_hist(PartIn in, u32* tile_counts) {
  __shared__ unsigned long long sh[2];
  const u64 ntiles = (in.n + BW_PART_TILE - 1) / BW_PART_TILE;
  for (u64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (threadIdx.x < 2) sh[threadIdx.x] = 0ULL;
    __syncthreads();
    // 8 destinations x 16-bit counters in two u64 (tile <= 2048 rows)
    unsigned long long c0 = 0, c1 = 0;
#pragma unroll
    for (int j = 0; j < BW_PART_PER_THREAD; ++j) {
      u64 i = tile * BW_PART_TILE + (u64)j * BW_PART_THREADS + threadIdx.x;
      if (i < in.n) {
        u32 d = bw_dest_of(bw_ld_stream_u64(in.keys + i), in.world);
        if (d < 4) c0 += 1ULL << (16 * d); else c1 += 1ULL << (16 * (d - 4));
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      c0 += __shfl_xor_sync(0xffffffffu, c0, o);
      c1 += __shfl_xor_sync(0xffffffffu, c1, o);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&sh[0], c0);
      atomicAdd(&sh[1], c1);
    }
    __syncthreads();
    if (threadIdx.x < BW_MAX_WORLD) {
      unsigned long long w = sh[threadIdx.x >> 2];
      tile_counts[tile * BW_MAX_WORLD + threadIdx.x] = (u32)((w >> (16 * (threadIdx.x & 3))) & 0xFFFFULL);
    }
    __syncthreads();
  }
}

// one block of 1024 threads per destination (grid = world); tile_counts -> exclusive offsets in place, totals published
__global__ void __launch_bounds__(1024) k_part_scan(u64 n, int world, u32* tile_counts, PartOut out, Counters* ctr) {
  __shared__ u32 strip[1024];
  const u64 ntiles = (n + BW_PART_TILE - 1) / BW_PART_TILE;
  const u64 per = (ntiles + blockDim.x - 1) / blockDim.x;
  const u64 lo = (u64)threadIdx.x * per, hi = (lo + per < ntiles) ? lo + per : ntiles;
  for (int d = blockIdx.x; d < world; d += gridDim.x) {
    u32 s = 0;
    for (u64 t = lo; t < hi; ++t) s += tile_counts[t * BW_MAX_WORLD + d];
    strip[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < (int)blockDim.x; o <<= 1) {
      u32 y = (threadIdx.x >= (unsigned)o) ? strip[threadIdx.x - o] : 0u;
      __syncthreads();
      strip[threadIdx.x] += y;
      __syncthreads();
    }
    u32 run = threadIdx.x ? strip[threadIdx.x - 1] : 0u;
    for (u64 t = lo; t < hi; ++t) {
      u32 c = tile_counts[t * BW_MAX_WORLD + d];
      tile_counts[t * BW_MAX_WORLD + d] = run;
      run += c;
    }
    if (threadIdx.x == blockDim.x - 1) {
      u64 total = strip[threadIdx.x];
      if (total > out.region_cap) bw_raise(ctr, 3u);
      *out.counts[d] = total;  // P2P: a store into rank d's memory
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) __threadfence_system();
}

// Stable scatter, staged through shared memory: rows of a tile are first laid out
// destination-major in shared memory, then every destination's run is copied out by the
// whole block with consecutive lanes on consecutive addresses.  Peer (NVLink) stores
// therefore arrive as long contiguous runs (2-8 KB per destination per tile) instead of
// warp-sized fragments -- the fragmented version reached ~200 GB/s over NVLink.
// SRC_ROW adds a fourth column, each row's index i in the source columns (u32), for an owner that must name the rows it
// received (K7 on N ranks); the dynamic shared memory then grows from BW_PART_TILE x 24 to BW_PART_TILE x 28 bytes.
// SIDE (with SRC_ROW) adds a fifth column, one byte per row from `side` (K8 on N ranks), and BW_PART_TILE more bytes of
// dynamic shared memory; without it `side` is not read.
template <bool SRC_ROW, bool SIDE = false>
__global__ void __launch_bounds__(BW_PART_THREADS)
k_part_scatter(PartIn in, const u32* tile_off, PartOut out, PartSide side) {
  static_assert(SRC_ROW || !SIDE, "the side column follows the source rows");
  // [iteration][warp][dest] counts, scanned in (iteration, warp) order per dest
  __shared__ u32 cnt[BW_PART_PER_THREAD][BW_PART_THREADS / 32][BW_MAX_WORLD];
  __shared__ u32 tot[BW_MAX_WORLD], dstart[BW_MAX_WORLD + 1];
  extern __shared__ __align__(16) unsigned char stage_raw[];
  u64* s_keys = (u64*)stage_raw;
  unsigned char* s_vals = stage_raw + (size_t)BW_PART_TILE * 8;
  i64* s_ts = (i64*)(s_vals + (size_t)BW_PART_TILE * (in.val_bytes ? in.val_bytes : 0));
  u32* s_row = (u32*)(s_ts + (in.ts ? BW_PART_TILE : 0));
  unsigned char* s_side = (unsigned char*)(s_row + BW_PART_TILE);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const u32 lt = (1u << lane) - 1u;
  const u64 ntiles = (in.n + BW_PART_TILE - 1) / BW_PART_TILE;
  for (u64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    u64 key[BW_PART_PER_THREAD];
    u32 dst[BW_PART_PER_THREAD], rk[BW_PART_PER_THREAD];
#pragma unroll
    for (int j = 0; j < BW_PART_PER_THREAD; ++j) {
      u64 i = tile * BW_PART_TILE + (u64)j * BW_PART_THREADS + threadIdx.x;
      bool valid = i < in.n;
      key[j] = valid ? bw_ld_stream_u64(in.keys + i) : 0ULL;
      dst[j] = valid ? bw_dest_of(key[j], in.world) : 0xFFu;
      rk[j] = 0;
#pragma unroll
      for (int d = 0; d < BW_MAX_WORLD; ++d) {
        u32 b = __ballot_sync(0xffffffffu, dst[j] == (u32)d);
        if (dst[j] == (u32)d) rk[j] = __popc(b & lt);
        if (lane == 0) cnt[j][warp][d] = __popc(b);
      }
    }
    __syncthreads();
    // warp d scans the 64 (iteration, warp) counters of destination d
    if (warp < BW_MAX_WORLD) {
      const int d = warp;
      u32 run = 0;
      for (int base = 0; base < BW_PART_PER_THREAD * (BW_PART_THREADS / 32); base += 32) {
        int e = base + lane;
        u32* p = &cnt[e / (BW_PART_THREADS / 32)][e % (BW_PART_THREADS / 32)][d];
        u32 v = *p, inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          u32 y = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += y;
        }
        *p = run + inc - v;
        run += __shfl_sync(0xffffffffu, inc, 31);
      }
      if (lane == 0) tot[d] = run;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      u32 acc = 0;
      for (int d = 0; d < BW_MAX_WORLD; ++d) {
        dstart[d] = acc;
        acc += tot[d];
      }
      dstart[BW_MAX_WORLD] = acc;
    }
    __syncthreads();
    // stage destination-major
#pragma unroll
    for (int j = 0; j < BW_PART_PER_THREAD; ++j) {
      u64 i = tile * BW_PART_TILE + (u64)j * BW_PART_THREADS + threadIdx.x;
      if (i < in.n) {
        const u32 d = dst[j];
        const u32 lp = dstart[d] + cnt[j][warp][d] + rk[j];
        s_keys[lp] = key[j];
        if (in.val_bytes == 8) {
          ((u64*)s_vals)[lp] = bw_ld_stream_u64((const u64*)in.vals + i);
        } else if (in.val_bytes == 4) {
          ((u32*)s_vals)[lp] = bw_ld_stream_u32((const u32*)in.vals + i);
        }
        if (in.ts) s_ts[lp] = (i64)bw_ld_stream_u64((const u64*)in.ts + i);
        if (SRC_ROW) s_row[lp] = (u32)i;
        if (SIDE) s_side[lp] = side.src[i];
      }
    }
    __syncthreads();
    // copy every destination's run out, block-wide, lane-consecutive
    for (int d = 0; d < in.world; ++d) {
      const u32 n_d = tot[d], s0 = dstart[d];
      const u64 g0 = tile_off[tile * BW_MAX_WORLD + d];
      u64* gk = out.keys[d] + g0;
      for (u32 e = threadIdx.x; e < n_d; e += BW_PART_THREADS) gk[e] = s_keys[s0 + e];
      if (in.val_bytes == 8) {
        u64* gv = (u64*)out.vals[d] + g0;
        for (u32 e = threadIdx.x; e < n_d; e += BW_PART_THREADS) gv[e] = ((const u64*)s_vals)[s0 + e];
      } else if (in.val_bytes == 4) {
        u32* gv = (u32*)out.vals[d] + g0;
        for (u32 e = threadIdx.x; e < n_d; e += BW_PART_THREADS) gv[e] = ((const u32*)s_vals)[s0 + e];
      }
      if (in.ts) {
        i64* gt = out.ts[d] + g0;
        for (u32 e = threadIdx.x; e < n_d; e += BW_PART_THREADS) gt[e] = s_ts[s0 + e];
      }
      if (SRC_ROW) {
        u32* gr = out.rows[d] + g0;
        for (u32 e = threadIdx.x; e < n_d; e += BW_PART_THREADS) gr[e] = s_row[s0 + e];
      }
      if (SIDE) {
        unsigned char* gs = side.dst[d] + g0;
        for (u32 e = threadIdx.x; e < n_d; e += BW_PART_THREADS) gs[e] = s_side[s0 + e];
      }
    }
    __syncthreads();
  }
}
// Instantiated here, before any kernel that declares its dynamic shared memory with a stricter alignment (bw_stream.cuh
// asks for 128 bytes): instantiated at the end of the translation unit, the staging would start at that alignment too.
template __global__ void k_part_scatter<false>(PartIn, const u32*, PartOut, PartSide);
template __global__ void k_part_scatter<true>(PartIn, const u32*, PartOut, PartSide);
template __global__ void k_part_scatter<true, true>(PartIn, const u32*, PartOut, PartSide);

// Keyed kernels on N ranks (K6, K7, K8; RankXchg in bwgpu.cu): what a source publishes beside its row count in every owner's
// region head, so that every owner can check that all ranks play the same call.  at[d] is this source's column in rank
// d's head; rows 1-3 of the head take the epoch, the system time and the refusal flag (row 0, the count, is
// k_part_scan's).
struct XchgHead {
  u64* at[BW_MAX_WORLD];
};
__global__ void k_xchg_head(XchgHead pub, int world, u64 epoch, i64 now, u64 refused) {
  if (threadIdx.x < (unsigned)world) {
    u64* h = pub.at[threadIdx.x];
    h[BW_MAX_WORLD] = epoch;
    h[2 * BW_MAX_WORLD] = (u64)now;
    h[3 * BW_MAX_WORLD] = refused;
  }
}

// A keyed map on N ranks (K5) returns each row's results to the rank that passed the row: the return section of one
// rank's region (RankXchg in bwgpu.cu), `cap` rows of mu, sigma and flag at the source's row index, and one error word
// per owner rank.
struct XchgRet {
  double* mu;
  double* sigma;
  unsigned char* flag;
  u32* err;  // [BW_MAX_WORLD]: owner rank d's table error (its t.err) after the call
};
struct XchgRetPeers {
  XchgRet at[BW_MAX_WORLD];  // every rank's return section as seen from this rank
};
