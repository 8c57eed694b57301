// bwgpu.cu -- libbwgpu.so: C ABI (include/bwgpu.h) over the sm_90a kernels.
//
// Host side of the epoch pump for ONE stateful step: what src/worker.rs:68-83
// (`Worker::run`) + src/operators.rs:667-1024 (one activation of
// `stateful_batch`) do per epoch, restated as stream-ordered kernel launches:
//
//   commit(epoch):  [H2D] -> (world>1: K1 partition + K2 exchange) -> prepass
//                   -> K3 fold (or the exact slow path) -> K4 close
//   advance():      wait, order rows like the reference, D2H
//   eof():          K4 over every key with watermark = UTC_MAX
//
// No torch, no Python: CUDA runtime + NCCL only.
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/bwgpu.h"
#include "bw_close.cuh"
#include "bw_common.cuh"
#include "bw_exchange.cuh"
#include "bw_stream.cuh"
#include "bw_snapshot.cuh"
#include "bw_fold.cuh"
#include "bw_keyed.cuh"
#include "bw_session.cuh"
#include "bw_jwin.cuh"
#include "bw_collect.cuh"
#include "bw_sjwin.cuh"
#include "bw_scwin.cuh"
#include "bw_argwin.cuh"
#include "bw_kcollect.cuh"
#include "bw_pjwin.cuh"
#include "bw_kjoin.cuh"
#include "bw_spjwin.cuh"
#include "bw_prepass.cuh"
#include "bw_slow.cuh"
#include "bw_late.cuh"

static thread_local std::string g_last_error;

// A "world" whose ranks are threads of ONE process on ONE GPU (bw_loopback_create): the collectives become host
// rendezvous + device-to-device copies and peer memory is plain pointers.  Every multi-rank code path -- routing
// hash, partition, exchange, combine / merge -- then runs on a single-GPU box (tests/test_gpu_loopback.py); the
// kernels and their arguments are the very same as over NCCL + CUDA IPC.
struct bw_loopback {
  int world = 0;
  std::mutex mu;
  std::condition_variable cv;
  int arrived = 0;
  unsigned long long generation = 0;
  const void* slot[BW_MAX_WORLD] = {nullptr};  // what each rank published for the collective in flight
  bool broken = false;
  // false when a peer thread never arrives (it failed and left): the world is then unusable, and says so
  bool barrier() {
    std::unique_lock<std::mutex> lk(mu);
    if (broken) return false;
    const unsigned long long g = generation;
    if (++arrived == world) {
      arrived = 0;
      ++generation;
      cv.notify_all();
      return true;
    }
    if (!cv.wait_for(lk, std::chrono::seconds(120), [&] { return generation != g || broken; }) || broken) {
      broken = true;
      cv.notify_all();
      return false;
    }
    return true;
  }
};

struct bw_ctx {
  int device = 0, rank = 0, world = 1, sm_count = BW_SM_COUNT_FALLBACK;
  ncclComm_t comm = nullptr;
  bw_loopback* loop = nullptr;
  std::string err;
  void* flush_buf = nullptr;
  size_t flush_bytes = 0;
};

#define CTX_FAIL(ctx, code, ...)                         \
  do {                                                   \
    char _b[512];                                        \
    snprintf(_b, sizeof _b, __VA_ARGS__);                \
    if (ctx) (ctx)->err = _b; else g_last_error = _b;    \
    return (code);                                       \
  } while (0)

#define CU(ctx, call)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      CTX_FAIL(ctx, BW_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, \
               __LINE__);                                                                          \
  } while (0)

#define NC(ctx, call)                                                                               \
  do {                                                                                              \
    ncclResult_t _e = (call);                                                                       \
    if (_e != ncclSuccess)                                                                          \
      CTX_FAIL(ctx, BW_ERR_NCCL, "%s failed: %s (%s:%d)", #call, ncclGetErrorString(_e), __FILE__,  \
               __LINE__);                                                                           \
  } while (0)

// Every CUDA resource of one native object (bw_fold, bw_smap, bw_join): device and pinned host memory, events and
// streams are made through it, and it releases them in reverse order when it goes.  A failed call leaves its field
// null.  regrow() frees a buffer before it allocates the new one, so peak memory does not rise, and a failure leaves
// the field null, never pointing at freed memory.
class Owner {
 public:
  enum Kind { DEV, HOST, EVENT, STREAM };
  Owner() = default;
  Owner(const Owner&) = delete;
  Owner& operator=(const Owner&) = delete;
  ~Owner() {
    for (size_t i = res_.size(); i-- > 0;) free_one(res_[i]);
  }
  // n elements of T (bytes when T is void), at least one
  template <typename T>
  cudaError_t dev(T** p, size_t n) { return mem(DEV, p, n); }
  template <typename T>
  cudaError_t host(T** p, size_t n) { return mem(HOST, p, n); }
  template <typename T>
  cudaError_t regrow(Kind k, T** p, size_t n) {
    release(*p);
    *p = nullptr;
    return mem(k, p, n);
  }
  cudaError_t event(cudaEvent_t* e, unsigned flags = cudaEventDisableTiming) {
    return keep(cudaEventCreateWithFlags(e, flags), EVENT, e);
  }
  cudaError_t stream(cudaStream_t* s, int priority = 0) {
    return keep(cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, priority), STREAM, s);
  }
  // release one resource made here before the object goes (null: nothing)
  void release(const void* h) {
    if (!h) return;
    for (size_t i = res_.size(); i-- > 0;)
      if (res_[i].h == h) {
        free_one(res_[i]);
        res_.erase(res_.begin() + i);
        return;
      }
  }

 private:
  struct Res {
    Kind kind;
    void* h;
  };
  std::vector<Res> res_;
  template <typename T>
  cudaError_t mem(Kind k, T** p, size_t n) {
    const size_t bytes = (n ? n : 1) * sizeof(std::conditional_t<std::is_void<T>::value, char, T>);
    void* q = nullptr;
    cudaError_t e = k == DEV ? cudaMalloc(&q, bytes) : cudaHostAlloc(&q, bytes, cudaHostAllocDefault);
    *p = (T*)q;
    return keep(e, k, p);
  }
  template <typename H>
  cudaError_t keep(cudaError_t e, Kind k, H* h) {
    if (e == cudaSuccess) res_.push_back({k, (void*)*h});
    else *h = nullptr;
    return e;
  }
  static void free_one(const Res& r) {
    switch (r.kind) {
      case DEV: cudaFree(r.h); break;
      case HOST: cudaFreeHost(r.h); break;
      case EVENT: cudaEventDestroy((cudaEvent_t)r.h); break;
      case STREAM: cudaStreamDestroy((cudaStream_t)r.h); break;
    }
  }
};

// ---- collectives: NCCL, or the loopback world's rendezvous ----
// all-gather of `bytes` per rank, device buffers, in stream order on `s`
static bw_status coll_allgather(bw_ctx* ctx, const void* send, void* recv, size_t bytes, cudaStream_t s) {
  if (!ctx->loop) {
    NC(ctx, ncclAllGather(send, recv, bytes, ncclChar, ctx->comm, s));
    return BW_OK;
  }
  bw_loopback* L = ctx->loop;
  CU(ctx, cudaStreamSynchronize(s));  // my contribution is complete
  L->slot[ctx->rank] = send;
  if (!L->barrier()) CTX_FAIL(ctx, BW_ERR_NCCL, "loopback world: a rank did not reach the all-gather");
  for (int r = 0; r < ctx->world; ++r)
    CU(ctx, cudaMemcpyAsync((char*)recv + (size_t)r * bytes, L->slot[r], bytes, cudaMemcpyDeviceToDevice, s));
  CU(ctx, cudaStreamSynchronize(s));
  // everyone has read everyone's buffer: it may be reused
  if (!L->barrier()) CTX_FAIL(ctx, BW_ERR_NCCL, "loopback world: a rank did not leave the all-gather");
  return BW_OK;
}
// barrier in stream order: completes on `s` once every rank's earlier work on its stream is done
static bw_status coll_barrier(bw_ctx* ctx, u32* d_word, cudaStream_t s) {
  if (!ctx->loop) {
    NC(ctx, ncclAllReduce(d_word, d_word, 1, ncclUint32, ncclMax, ctx->comm, s));
    return BW_OK;
  }
  CU(ctx, cudaStreamSynchronize(s));
  if (!ctx->loop->barrier()) CTX_FAIL(ctx, BW_ERR_NCCL, "loopback world: a rank did not reach the barrier");
  return BW_OK;
}
// every rank's `base` pointer as seen from this rank (CUDA IPC mappings, or the pointers themselves)
static bw_status coll_share_base(bw_ctx* ctx, void* base, void** peers, cudaStream_t s) {
  const int W = ctx->world;
  if (ctx->loop) {
    bw_loopback* L = ctx->loop;
    L->slot[ctx->rank] = base;
    if (!L->barrier()) CTX_FAIL(ctx, BW_ERR_NCCL, "loopback world: a rank did not publish its buffer");
    for (int r = 0; r < W; ++r) peers[r] = const_cast<void*>(L->slot[r]);
    if (!L->barrier()) CTX_FAIL(ctx, BW_ERR_NCCL, "loopback world: a rank did not read the buffers");
    return BW_OK;
  }
  cudaIpcMemHandle_t mine;
  CU(ctx, cudaIpcGetMemHandle(&mine, base));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
  unsigned char *d_in = nullptr, *d_all = nullptr;
  Owner tmp;  // the two staging buffers, freed on every way out
  CU(ctx, tmp.dev(&d_in, 64));
  CU(ctx, tmp.dev(&d_all, 64 * W));
  CU(ctx, cudaMemcpy(d_in, &mine, 64, cudaMemcpyHostToDevice));
  NC(ctx, ncclAllGather(d_in, d_all, 64, ncclChar, ctx->comm, s));
  CU(ctx, cudaStreamSynchronize(s));
  std::vector<cudaIpcMemHandle_t> all(W);
  CU(ctx, cudaMemcpy(all.data(), d_all, 64 * W, cudaMemcpyDeviceToHost));
  for (int r = 0; r < W; ++r) {
    if (r == ctx->rank) peers[r] = base;
    else CU(ctx, cudaIpcOpenMemHandle(&peers[r], all[r], cudaIpcMemLazyEnablePeerAccess));
  }
  return BW_OK;
}

struct Slot {
  u64* h_keys = nullptr;
  void* h_vals = nullptr;
  i64* h_ts = nullptr;
  bool acquired = false;
};
struct Stage {  // device staging for host-ingested batches
  u64* d_keys = nullptr;
  void* d_vals = nullptr;
  i64* d_ts = nullptr;
  cudaEvent_t consumed = nullptr;  // recorded after the kernels that read it
  bool used = false;
};

struct EventPair {
  cudaEvent_t a, b;
  u64 rows;
  int kind;  // 0: fold stage (k_fold / k_segfold), 1: k_scatter, 2: k_verdict
};

typedef void (*scatter_kernel_t)(ScatterArgs, FoldParams);
typedef void (*segfold_kernel_t)(SegArgs, Table, FoldParams, EmitBufs);

// Scratch of the reference-order permutation (order_perm): sort keys, the permutation, one gathered column and CUB's
// temporary storage.
struct SortScratch {
  u64 cap = 0;
  u64 *sk = nullptr, *sk2 = nullptr, *gather = nullptr;
  u32 *perm = nullptr, *perm2 = nullptr;
  void* cub = nullptr;
  size_t cub_bytes = 0;
  // room for n rows: when they do not fit, reallocate for grow_to (>= n) rows once nothing on `s` reads the old buffers
  cudaError_t reserve(Owner& own, u64 n, u64 grow_to, cudaStream_t s) {
    if (n <= cap) return cudaSuccess;
    cudaError_t e = cudaStreamSynchronize(s);
    cap = 0;
    for (u64** p : {&sk, &sk2, &gather})
      if (!e) e = own.regrow(Owner::DEV, p, grow_to);
    for (u32** p : {&perm, &perm2})
      if (!e) e = own.regrow(Owner::DEV, p, grow_to);
    if (e) return e;
    size_t b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b, sk, sk2, perm, perm2, (int)grow_to, 0, 64, s);
    if ((e = grow_cub(own, b + 256))) return e;
    cap = grow_to;
    return cudaSuccess;
  }
  // CUB's temporary storage: at least `bytes`, never shrunk
  cudaError_t grow_cub(Owner& own, size_t bytes) {
    if (bytes <= cub_bytes) return cudaSuccess;
    cub_bytes = 0;
    cudaError_t e = own.regrow(Owner::DEV, &cub, bytes);
    if (!e) cub_bytes = bytes;
    return e;
  }
};

// Five pinned host columns of 8-byte values, grown together: the rows an advance hands to the caller.
struct HostCols {
  u64 cap = 0;
  u64* col[5] = {};
  cudaError_t reserve(Owner& own, u64 n, u64 grow_to) {
    if (n <= cap) return cudaSuccess;
    cap = 0;
    for (u64*& c : col)
      if (cudaError_t e = own.regrow(Owner::HOST, &c, grow_to)) return e;
    cap = grow_to;
    return cudaSuccess;
  }
};

struct Stage;
// An activation whose scatter + verdict are queued but whose fold stage is not: the host looks at a
// verdict only after the NEXT activation's scatter is queued, so the device never waits for the host.
struct Deferred {
  bool valid = false;
  int side = 0;
  const u64* d_keys = nullptr;
  const void* d_vals = nullptr;
  const i64* d_ts = nullptr;
  u64 rows = 0, ord = 0;
  u32 batch_no = 0;
  u32 lanes = 0;           // blocks of this activation's scatter
  Stage* stage = nullptr;  // device staging buffer to release once the fold has read it
};

struct bw_fold {
  Owner own;  // every buffer, event and stream below
  bw_ctx* ctx = nullptr;
  bw_fold_spec spec{};
  FoldParams p{};
  Table t{};
  int force_seg_shift = -1;  // env BW_SEG_SHIFT: t.seg_shift in place of BW_SEG_SHIFT_DEFAULT (-1: not set)
  u32 segfold_parts = BW_SF_ALL;  // BW_SF_*: bw_fold_set_segfold_parts measures what each part of the segment fold is worth
  EmitBufs e{};
  Counters* d_ctr = nullptr;
  Counters* h_ctr = nullptr;  // pinned mirror
  cudaStream_t s_compute = nullptr, s_copy = nullptr, s_pre = nullptr, s_x = nullptr;  // s_x: partition + exchange
  cudaEvent_t ev_fold_done = nullptr, ev_xchg_done = nullptr;
  bool fold_recorded = false;
  cudaEvent_t ev_gen = nullptr;      // last bw_gen_c1 (the only producer of device columns this library runs itself)
  // the columns of the activation in flight are complete once this has happened (null: nothing to wait for); the
  // lateness pass on s_pre and the exchange on s_x wait on it
  cudaEvent_t cols_ready = nullptr;
  cudaEvent_t ev_pre = nullptr, ev_h2d = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  int val_bytes = 8;
  bool has_vals = true, has_ts = false;
  // ingest
  std::vector<Slot> slots;
  std::vector<Stage> stages;
  u32 stage_next = 0;
  // prepass
  i64 *d_rmin = nullptr, *d_rmax = nullptr;
  u32* d_rbad = nullptr;
  u32* h_verdict = nullptr;  // pinned
  u32* d_verdict = nullptr;
  u64 max_recv_rows = 0;
  // slow path temp (lazy)
  u64 slow_cap = 0;
  u64 *d_kflat = nullptr, *d_ksorted = nullptr;
  i64 *d_tsflat = nullptr, *d_tssorted = nullptr, *d_prefmax = nullptr;
  u32 *d_idx = nullptr, *d_idxsorted = nullptr;
  unsigned char* d_late = nullptr;
  // emission ordering scratch, sized at create; the slow path shares its CUB storage
  SortScratch srt;
  // Rows of CLOSED epochs are ordered and copied to the host while later activations run (side stream s_out, its own
  // sort scratch): bw_advance then only has the newest rows left to do.  One rank, see flush_rows().
  SortScratch fl;
  struct RowMark {
    u64 epoch = 0, next_epoch = 0;  // next_epoch: 1 + epoch of the activation folded after this one (0: none yet)
    cudaEvent_t ev = nullptr;       // the counts below are on the host once this has happened
    bool live = false;
  } marks[4];
  unsigned long long* h_marks = nullptr;  // pinned [4][2]: n_closed, n_late after the marked activation
  u32 mark_head = 0;                      // marks enqueued so far
  u64 done_c = 0, done_l = 0;             // rows already ordered and on the host
  cudaStream_t s_out = nullptr;
  u32 timer_stride = 4;                   // env BW_TIMER_STRIDE: every n-th activation's kernels are timed with CUDA events
  bool flush_on = true;                   // env BW_FLUSH=0: order and copy everything in bw_advance
  bool host_ingest = false;               // the caller commits HOST batches (PCIe-bound: the device has time to spare between
                                          // activations; a device-resident caller keeps every SM busy and is left alone)
  // host output (pinned, grown on demand): closed {key, window id, acc, count, epoch}, late {key, window id, value,
  // timestamp, epoch}
  HostCols ho_c, ho_l;
  // bookkeeping
  u32 batch_no = 0;
  u64 last_epoch = 0, min_epoch = 0;  // epochs are non-decreasing; rows carry the user epoch
  bool have_epoch = false, have_pending = false;
  bool eof_done = false;
  int fold_grid = 0, close_grid = 0;
  void (*fold_kernel)(BatchView, Table, FoldParams, u32, u32, u32) = nullptr;
  // streaming fold (bw_stream.cuh): fused verdict + bucket scatter, shared-memory segment fold
  StreamBufs sb{};
  bool stream_ok = false;   // buffers allocated, fold type supported
  int stream_mode = 1;      // env BW_STREAM=0: always take the direct kernel (k_fold)
  int scatter_grid = 0, segfold_grid = 0;
  scatter_kernel_t scatter_kernel = nullptr;
  segfold_kernel_t segfold_kernel = nullptr;
  size_t segfold_smem = 0, scatter_smem = 0;
  int scatter_nstage = 3;
  u32 last_scatter_grid = 0, scatter_stg_cap = 0, scatter_stg_every = 1, scatter_ovf_cap = 0;
  // env BW_SC_STG / BW_SC_EVERY / BW_SC_STAGES: the three above, in place of what stream_alloc picks for the shape (-1: not set)
  int force_stg_cap = -1, force_stg_every = -1, force_nstage = -1;
  // multi-GPU streaming path: combine at the source, partials over NVLink, merge at the owner
  segfold_kernel_t combine_kernel = nullptr, merge_kernel = nullptr;
  int combine_grid = 0, merge_grid = 0;
  u32 nb_local = 0, part_cap = 0;
  void* precv_base = nullptr;            // this rank's receive regions (IPC-shared): [side]{cnt[W][nb_local], rec[W][nb_local][part_cap]}
  void* precv_peer[BW_MAX_WORLD] = {nullptr};
  size_t precv_cnt_off[2] = {0, 0}, precv_rec_off[2] = {0, 0};
  VerdictGather* d_vg_local = nullptr;   // [2]
  VerdictGather* d_vg_all = nullptr;     // [2][W]
  VerdictGather* h_vg = nullptr;         // pinned [2][W]
  bool vg_pending[2] = {false, false};   // a side's local verdict is computed but not gathered yet
  cudaEvent_t ev_vg[2] = {nullptr, nullptr};
  i64 h_gmax = INT64_MIN;                // running maximum event time over all ranks (the verdict chain's memory)
  u32* d_barrier_word = nullptr;
  cudaEvent_t ev_sv[2] = {nullptr, nullptr};
  StreamVerdict* h_sv = nullptr;  // pinned mirror of the two sides' verdicts
  // activations with a few late rows (bw_late.cuh); buffers are made on first use
  LateBufs late = {};
  bool late_ready = false;
  bool late_split = true;   // env BW_LATE_SPLIT=0: every not-clean activation takes the sort path
  u32* h_late_ctr = nullptr;  // pinned: suspects seen, table overflow
  i64* late_chunk_pre = nullptr;  // [tiles][32] running maximum before every 64-row chunk
  Deferred dq{};            // the activation whose fold has not been launched yet
  i64* d_span = nullptr;   // [min ts, max ts] of the activation (prepass)
  // snapshot staging (bw_snapshot_take, bw_snapshot_load)
  void* snap_dev = nullptr;
  void* snap_host = nullptr;
  unsigned long long* d_snap_ctr = nullptr;
  // multi-GPU exchange
  void* xchg_base = nullptr;  // one allocation, IPC-shared
  size_t xchg_bytes = 0;
  void* peer_base[BW_MAX_WORLD] = {nullptr};
  u64 region_cap = 0;
  u32* d_tile_counts = nullptr;
  u64* d_send_counts = nullptr;   // NCCL mode
  u64* d_all_counts = nullptr;    // NCCL mode [world][world]
  u64* h_all_counts = nullptr;    // pinned
  u64 *send_keys = nullptr;       // NCCL mode local send regions
  void* send_vals = nullptr;
  i64* send_ts = nullptr;
  int xbuf = 0;
  // stats
  bw_stats st{};
  std::vector<EventPair> timers;
  size_t timers_used = 0;
};

#define FAIL(f, code, ...) CTX_FAIL((f)->ctx, code, __VA_ARGS__)
static bw_status mark_rows(bw_fold* f, u64 epoch);
static bw_status flush_rows(bw_fold* f);

// ---------------------------------------------------------------------------
// small kernels
// ---------------------------------------------------------------------------
__global__ void k_init_table(Table t, u64 acc_identity) {
  const u64 n = t.cap + 1;
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (u64)gridDim.x * blockDim.x) {
    HotSlot h;
    bw_key_put(t, h, s, BW_EMPTY_KEY);
    h.max_ts = INT64_MIN;
    h.wt0 = BW_EMPTY_WIDTAG;
    h.acc0 = acc_identity;
    t.hot[s] = h;
    P1Slot c;
    c.acc1 = acc_identity;
    c.seq1 = ~0ULL;
    t.p1[s] = c;
    AuxSlot x;
    x.seq0 = ~0ULL;
    x.cnt0 = 0;
    x.cnt1 = 0;
    x.spill_head = 0;
    x.lock = 0;
    t.aux[s] = x;
    t.closed_upto[s] = INT64_MIN;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    Counters z;
    memset(&z, 0, sizeof z);
    z.pool_next = 1;  // node 0 is the null node
    z.gmax_ts = (unsigned long long)INT64_MIN;
    *t.ctr = z;
  }
}

__global__ void k_gen_c1(u64* keys, u64* vals, u64 start, u64 rows, u64 n_keys) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (u64)gridDim.x * blockDim.x) {
    u64 g = start + i;
    keys[i] = bw_splitmix64(0x5EEDULL ^ g) % n_keys;
    vals[i] = g;
  }
}

__global__ void k_fill(unsigned char* p, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n / 16; i += (size_t)gridDim.x * blockDim.x)
    ((uint4*)p)[i] = make_uint4(0xA5A5A5A5u, 0xA5A5A5A5u, 0xA5A5A5A5u, 0xA5A5A5A5u);
}

// ---------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------
// (C linkage comes from the declarations in include/bwgpu.h)

uint32_t bw_abi_version(void) { return BW_ABI_VERSION; }
const char* bw_last_global_error(void) { return g_last_error.c_str(); }
const char* bw_last_error(const bw_ctx* ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }

uint32_t bw_route(uint64_t key, uint32_t world) { return bw_route_hash(bw_mix64(key), world); }

bw_status bw_nccl_unique_id(void* out128) {
  ncclUniqueId id;
  ncclResult_t r = ncclGetUniqueId(&id);
  if (r != ncclSuccess) {
    g_last_error = std::string("ncclGetUniqueId failed: ") + ncclGetErrorString(r);
    return BW_ERR_NCCL;
  }
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  memcpy(out128, &id, 128);
  return BW_OK;
}

bw_status bw_ctx_create(int device, int rank, int world, const void* nccl_unique_id, bw_ctx** out) {
  bw_ctx* null_ctx = nullptr;
  if (!out) CTX_FAIL(null_ctx, BW_ERR_SPEC, "bw_ctx_create: out is NULL");
  if (world < 1 || world > BW_MAX_WORLD || rank < 0 || rank >= world)
    CTX_FAIL(null_ctx, BW_ERR_SPEC, "bw_ctx_create: bad rank/world %d/%d (max world %d)", rank, world, BW_MAX_WORLD);
  if (world > 1 && !nccl_unique_id) CTX_FAIL(null_ctx, BW_ERR_SPEC, "bw_ctx_create: world > 1 needs an NCCL id");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev <= 0)
    CTX_FAIL(null_ctx, BW_ERR_CUDA, "no CUDA device: %s", cudaGetErrorString(ce));
  if (device < 0 || device >= ndev) CTX_FAIL(null_ctx, BW_ERR_SPEC, "device %d out of range (%d devices)", device, ndev);
  CU(null_ctx, cudaSetDevice(device));
  cudaDeviceProp prop;
  CU(null_ctx, cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)  // sm_90a code runs on compute capability 9.0 only
    CTX_FAIL(null_ctx, BW_ERR_CUDA, "libbwgpu is built for sm_90a only; device %d is sm_%d%d", device, prop.major,
             prop.minor);
  bw_ctx* c = new bw_ctx();
  c->device = device;
  c->rank = rank;
  c->world = world;
  c->sm_count = prop.multiProcessorCount;
  if (world > 1) {
    ncclUniqueId id;
    memcpy(&id, nccl_unique_id, 128);
    ncclResult_t r = ncclCommInitRank(&c->comm, world, id, rank);
    if (r != ncclSuccess) {
      g_last_error = std::string("ncclCommInitRank failed: ") + ncclGetErrorString(r);
      delete c;
      return BW_ERR_NCCL;
    }
  }
  *out = c;
  return BW_OK;
}

bw_status bw_loopback_create(int world, bw_loopback** out) {
  bw_ctx* null_ctx = nullptr;
  if (!out || world < 2 || world > BW_MAX_WORLD) CTX_FAIL(null_ctx, BW_ERR_SPEC, "bw_loopback_create: world must be in 2..%d", BW_MAX_WORLD);
  bw_loopback* L = new bw_loopback();
  L->world = world;
  *out = L;
  return BW_OK;
}
void bw_loopback_destroy(bw_loopback* world) { delete world; }

bw_status bw_ctx_create_loopback(int device, int rank, bw_loopback* world, bw_ctx** out) {
  bw_ctx* null_ctx = nullptr;
  if (!out || !world || rank < 0 || rank >= world->world) CTX_FAIL(null_ctx, BW_ERR_SPEC, "bw_ctx_create_loopback: bad arguments");
  bw_ctx* c = nullptr;
  bw_status st = bw_ctx_create(device, 0, 1, nullptr, &c);  // device checks; no communicator
  if (st != BW_OK) return st;
  c->rank = rank;
  c->world = world->world;
  c->loop = world;
  *out = c;
  return BW_OK;
}

void bw_ctx_destroy(bw_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->comm) ncclCommDestroy(ctx->comm);
  if (ctx->flush_buf) cudaFree(ctx->flush_buf);
  delete ctx;
}

bw_status bw_dev_alloc(bw_ctx* ctx, uint64_t bytes, void** out) {
  CU(ctx, cudaSetDevice(ctx->device));
  CU(ctx, cudaMalloc(out, bytes ? bytes : 16));
  return BW_OK;
}
bw_status bw_dev_free(bw_ctx* ctx, void* ptr) {
  CU(ctx, cudaFree(ptr));
  return BW_OK;
}
bw_status bw_host_alloc(bw_ctx* ctx, uint64_t bytes, void** out) {
  CU(ctx, cudaSetDevice(ctx->device));
  CU(ctx, cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocDefault));
  return BW_OK;
}
bw_status bw_host_free(bw_ctx* ctx, void* ptr) {
  CU(ctx, cudaFreeHost(ptr));
  return BW_OK;
}
bw_status bw_memcpy(bw_ctx* ctx, void* dst, const void* src, uint64_t bytes, int kind) {
  cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  CU(ctx, cudaMemcpy(dst, src, bytes, k));
  return BW_OK;
}
bw_status bw_flush_l2(bw_ctx* ctx) {
  CU(ctx, cudaSetDevice(ctx->device));
  if (!ctx->flush_buf) {
    ctx->flush_bytes = (size_t)256 << 20;  // 256 MiB > 50 MB L2
    CU(ctx, cudaMalloc(&ctx->flush_buf, ctx->flush_bytes));
  }
  k_fill<<<ctx->sm_count * 8, 256>>>((unsigned char*)ctx->flush_buf, ctx->flush_bytes);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaDeviceSynchronize());
  return BW_OK;
}

// ---------------------------------------------------------------------------
// fold create / destroy
// ---------------------------------------------------------------------------
static i64 gcd_i64(i64 a, i64 b) {
  while (b) {
    i64 t = a % b;
    a = b;
    b = t;
  }
  return a;
}

// k_fold instantiations: accumulator op x watermark tracking (+ MEAN keeps counts)
typedef void (*fold_kernel_t)(BatchView, Table, FoldParams, u32, u32, u32);
template <int OP, int CNT>
static fold_kernel_t pick_wm(bool wm) {
  return wm ? (fold_kernel_t)k_fold<FoldCfg<OP, 1, CNT>> : (fold_kernel_t)k_fold<FoldCfg<OP, 0, CNT>>;
}
static fold_kernel_t pick_fold_kernel(const FoldParams& p) {
  const bool wm = p.track_wm != 0;
  if (p.need_count) return pick_wm<BW_OP_ADD_F64, 1>(wm);
  switch (p.op) {
    case BW_OP_ADD_ONE: return pick_wm<BW_OP_ADD_ONE, 0>(wm);
    case BW_OP_ADD_U64: return pick_wm<BW_OP_ADD_U64, 0>(wm);
    case BW_OP_ADD_F64: return pick_wm<BW_OP_ADD_F64, 0>(wm);
    case BW_OP_MIN_S64: return pick_wm<BW_OP_MIN_S64, 0>(wm);
    case BW_OP_MIN_U64: return pick_wm<BW_OP_MIN_U64, 0>(wm);
    case BW_OP_MAX_S64: return pick_wm<BW_OP_MAX_S64, 0>(wm);
    default: return pick_wm<BW_OP_MAX_U64, 0>(wm);
  }
}

// k_segfold instantiations: accumulator op (+ counts for MEAN) x first-open indices
template <int OP, int CNT, int MODE>
static segfold_kernel_t pick_seq(bool seq) {
  return seq ? (segfold_kernel_t)k_segfold<FoldCfg<OP, -1, CNT>, true, MODE> : (segfold_kernel_t)k_segfold<FoldCfg<OP, -1, CNT>, false, MODE>;
}
// MODE: 0 one GPU, 1 combine at the source rank, 2 merge at the owning rank (bw_stream.cuh)
template <int MODE>
static segfold_kernel_t pick_segfold_kernel(const FoldParams& p) {
  const bool seq = !p.seq_by_id;
  if (p.need_count) return pick_seq<BW_OP_ADD_F64, 1, MODE>(seq);
  switch (p.op) {
    case BW_OP_ADD_ONE: return pick_seq<BW_OP_ADD_ONE, 0, MODE>(seq);
    case BW_OP_ADD_U64: return pick_seq<BW_OP_ADD_U64, 0, MODE>(seq);
    case BW_OP_ADD_F64: return pick_seq<BW_OP_ADD_F64, 0, MODE>(seq);
    case BW_OP_MIN_S64: return pick_seq<BW_OP_MIN_S64, 0, MODE>(seq);
    case BW_OP_MIN_U64: return pick_seq<BW_OP_MIN_U64, 0, MODE>(seq);
    case BW_OP_MAX_S64: return pick_seq<BW_OP_MAX_S64, 0, MODE>(seq);
    default: return pick_seq<BW_OP_MAX_U64, 0, MODE>(seq);
  }
}
// k_scatter instantiations: timestamp source x value bytes read / stored
static scatter_kernel_t pick_scatter_kernel(int tsm, int vb_in, int vb_out) {
  if (tsm == 1) return vb_out ? (scatter_kernel_t)k_scatter<1, 8, 8> : (scatter_kernel_t)k_scatter<1, 8, 0>;
  if (tsm == 0) {
    if (!vb_out) return (scatter_kernel_t)k_scatter<0, 0, 0>;
    return vb_in == 4 ? (scatter_kernel_t)k_scatter<0, 4, 4> : (scatter_kernel_t)k_scatter<0, 8, 8>;
  }
  if (!vb_out) return (scatter_kernel_t)k_scatter<2, 0, 0>;
  return vb_in == 4 ? (scatter_kernel_t)k_scatter<2, 4, 4> : (scatter_kernel_t)k_scatter<2, 8, 8>;
}

static bw_status stream_alloc(bw_fold* f) {
  bw_ctx* ctx = f->ctx;
  Owner& own = f->own;
  StreamBufs& sb = f->sb;
  const u64 rows = f->spec.max_batch_rows;
  const int W = ctx->world;
  f->nb_local = (u32)(f->t.cap >> f->t.seg_shift);
  const u64 nb = (u64)f->nb_local * W;  // buckets of the scatter: (owning rank, segment of its table)
  if (!f->stream_mode || nb > BW_STREAM_MAX_NB || rows >= (1ULL << 28)) return BW_OK;
  if (W > 1 && f->spec.exchange != BW_XCHG_P2P) return BW_OK;  // the partials travel as peer stores
  // wait == forever with event time: nothing closes before EOF, every key grows an overflow list of panes --
  // the shape the direct kernel's general path is for
  if (!f->p.track_wm && f->p.ts_from_value != 2) return BW_OK;
  sb.nb = (u32)nb;
  // Every scatter block owns a lane in every bucket's region.  A lane holds the block's share of the bucket's rows: mean
  // + 6 sigma, where the variance is that of the rows (Poisson) plus that of the bucket's number of distinct keys (a fuller
  // lane overflows into the spill list).
  sb.nlanes = (u32)ctx->sm_count;
  const u64 max_tiles = (rows + BW_SC_TILE - 1) / BW_SC_TILE;
  const double block_rows = (double)((max_tiles + sb.nlanes - 1) / sb.nlanes) * BW_SC_TILE;
  const double mean = block_rows / (double)nb;
  const double keys_per_bucket = std::max(1.0, (double)std::max<u64>(f->spec.capacity_hint, 1) / (double)f->nb_local);
  const double sigma = std::sqrt(mean + mean * mean / keys_per_bucket);
  sb.lane_cap = (u32)std::min<double>(block_rows, mean + 6.0 * sigma + 24.0);
  sb.lane_cap = (sb.lane_cap + 7u) & ~7u;
  // every row can end up there in the worst case (a pane per event beyond a key's two direct panes: sparse sliding folds)
  sb.spill_cap = (u32)std::min<u64>(std::max<u64>(rows + rows / 8, 8192), 1u << 26);
  sb.val_bytes = (f->p.op == BW_OP_ADD_ONE && !f->p.need_count) ? 0 : f->val_bytes;
  const size_t region_rows = (size_t)sb.nb * sb.nlanes * sb.lane_cap;
  for (int i = 0; i < 2; ++i) {
    CU(ctx, own.dev(&sb.side[i].rec, region_rows));
    if (sb.val_bytes) CU(ctx, own.dev(&sb.side[i].val, region_rows * (size_t)sb.val_bytes));
    CU(ctx, own.dev(&sb.side[i].cnt, (size_t)sb.nb * sb.nlanes));
    CU(ctx, cudaMemsetAsync(sb.side[i].cnt, 0, sizeof(u32) * sb.nb * sb.nlanes, f->s_compute));
    CU(ctx, own.dev(&sb.side[i].spill, sb.spill_cap));
    CU(ctx, own.dev(&sb.side[i].sv, 1));
    CU(ctx, cudaMemsetAsync(sb.side[i].sv, 0, sizeof(StreamVerdict), f->s_compute));
    CU(ctx, own.event(&f->ev_sv[i]));
  }
  CU(ctx, own.host(&f->h_sv, 2));
  const int tsm = f->p.ts_from_value ? f->p.ts_from_value : 0;
  const int vb_in = (tsm == 1) ? 8 : (sb.val_bytes ? f->val_bytes : 0);
  f->scatter_kernel = pick_scatter_kernel(tsm, vb_in, sb.val_bytes);
  sb.tiles_cap = (u32)((rows + BW_SC_TILE - 1) / BW_SC_TILE + 1);  // one lateness triple per scatter tile
  // (one set per side: the tile triples of activation b are read again when it turns out to have late rows, after the
  // scatter of b + 1 has run)
  CU(ctx, own.dev(&sb.tile_min, 2 * (size_t)sb.tiles_cap));
  CU(ctx, own.dev(&sb.tile_max, 2 * (size_t)sb.tiles_cap));
  CU(ctx, own.dev(&sb.tile_bad, 2 * (size_t)sb.tiles_cap));
  CU(ctx, own.dev(&sb.chunk_max, 2 * (size_t)sb.tiles_cap * BW_SC_WARPS));
  // Shared memory of the scatter: up to 16 records per bucket assembled before they are written out (counts only: the
  // value column is not staged), then as many TMA stages of the input tile (2..4) as still fit.  Deeper staging beats
  // more stages: on C1 (489 buckets; H100 SXM, 700 W) 16 records with 2 stages take 0.233 ms, 8 records with 4 stages
  // 0.318 ms -- fewer, longer runs of a lane's 128-byte lines written per write-out, and a third as many write-outs.
  const size_t smem_budget = 208 * 1024;
  f->scatter_stg_cap = 0;
  if (sb.val_bytes == 0)
    for (u32 c : {16u, 8u, 6u, 4u})
      if (bw_scatter_smem(tsm, vb_in, 2, sb.nb, c, 0) <= smem_budget) {
        f->scatter_stg_cap = c;
        break;
      }
  if (f->force_stg_cap >= 0) f->scatter_stg_cap = (u32)f->force_stg_cap;
  // write out when an average bucket has assembled ~7/8 of its staging rows, half a row of which on average is the odd
  // row the last write-out left behind (C1 on an H100 SXM, 700 W, 16 records: every tile 0.295 ms, every 2 tiles 0.244,
  // every 3 -- this rule's choice -- 0.233)
  const double fill_tiles = 0.875 * std::max(0.0, f->scatter_stg_cap - 0.5) * (double)sb.nb / BW_SC_TILE;
  f->scatter_stg_every = (u32)std::max<double>(1.0, std::floor(fill_tiles));
  if (f->force_stg_every >= 0) f->scatter_stg_every = (u32)f->force_stg_every;
  f->scatter_nstage = 4;
  while (f->scatter_nstage > 2 && bw_scatter_smem(tsm, vb_in, f->scatter_nstage, sb.nb, f->scatter_stg_cap, 0) > smem_budget) --f->scatter_nstage;
  if (f->force_nstage >= 0) f->scatter_nstage = f->force_nstage;
  if (bw_scatter_smem(tsm, vb_in, f->scatter_nstage, sb.nb, f->scatter_stg_cap, 0) > 216 * 1024) return BW_OK;  // too many segments
  // rows that outrun their bucket's staging rows wait in what the budget leaves, up to 1024 of them (C1: ~170 per
  // write-out on average, from a Poisson count of mean 12.6 against 16 staging rows).  Not when a tile alone outruns an
  // average bucket's staging: most rows would then pass through the area, all on one shared-memory counter (10^5 keys,
  // 49 buckets: 0.307 ms with the area against 0.292 without, same card)
  f->scatter_ovf_cap = 0;
  if (f->scatter_stg_cap && fill_tiles >= 1.0) {
    const size_t used = bw_scatter_smem(tsm, vb_in, f->scatter_nstage, sb.nb, f->scatter_stg_cap, 0);
    if (used < smem_budget) f->scatter_ovf_cap = (u32)std::min<size_t>(1024, (smem_budget - used) / 24) & ~31u;
  }
  f->scatter_smem = bw_scatter_smem(tsm, vb_in, f->scatter_nstage, sb.nb, f->scatter_stg_cap, f->scatter_ovf_cap);
  // the attribute belongs to the kernel, not to this fold: folds with other table sizes share it
  CU(ctx, cudaFuncSetAttribute((const void*)f->scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));
  int occ = 0;
  CU(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)f->scatter_kernel, BW_SC_THREADS, f->scatter_smem));
  f->scatter_grid = ctx->sm_count * std::max(occ, 1);
  f->segfold_kernel = pick_segfold_kernel<0>(f->p);
  f->segfold_smem = bw_segfold_smem(1u << f->t.seg_shift, f->p.op, !f->p.seq_by_id, f->p.need_count != 0);
  CU(ctx, cudaFuncSetAttribute((const void*)f->segfold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));
  CU(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)f->segfold_kernel, BW_SF_THREADS, f->segfold_smem));
  f->segfold_grid = ctx->sm_count * std::max(occ, 1);
  if (W > 1) {
    f->combine_kernel = pick_segfold_kernel<1>(f->p);
    f->merge_kernel = pick_segfold_kernel<2>(f->p);
    for (segfold_kernel_t k : {f->combine_kernel, f->merge_kernel}) {
      CU(ctx, cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));
      CU(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)k, BW_SF_THREADS, f->segfold_smem));
      (k == f->combine_kernel ? f->combine_grid : f->merge_grid) = ctx->sm_count * std::max(occ, 1);
    }
    // receive regions: a source can leave at most two partials (two panes) per slot of a segment
    f->part_cap = 2u << f->t.seg_shift;
    size_t off = 0;
    auto take = [&](size_t bytes) {
      size_t o = off;
      off += (bytes + 255) & ~(size_t)255;
      return o;
    };
    for (int sd = 0; sd < 2; ++sd) {
      f->precv_cnt_off[sd] = take(sizeof(u32) * (size_t)W * f->nb_local);
      f->precv_rec_off[sd] = take(sizeof(Partial) * (size_t)W * f->nb_local * f->part_cap);
    }
    CU(ctx, own.dev(&f->precv_base, off));
    CU(ctx, cudaMemset(f->precv_base, 0, off));
    {
      bw_status cst = coll_share_base(ctx, f->precv_base, f->precv_peer, f->s_compute);
      if (cst != BW_OK) return cst;
    }
    CU(ctx, own.dev(&f->d_vg_local, 2));
    CU(ctx, own.dev(&f->d_vg_all, 2 * (size_t)W));
    CU(ctx, own.host(&f->h_vg, 2 * (size_t)W));
    CU(ctx, own.dev(&f->d_barrier_word, 1));
    CU(ctx, cudaMemset(f->d_barrier_word, 0, 4));
    // the legacy path is now the fallback of single activations: it runs in line with the rest (its own stream only
    // bought overlap between consecutive legacy activations, and its lateness pass must see the maximum set here)
    if (f->s_x && f->s_x != f->s_compute) {
      own.release(f->s_x);
      f->s_x = f->s_compute;
    }
  }
  f->stream_ok = true;
  return BW_OK;
}

static bw_status fold_alloc(bw_fold* f) {
  bw_ctx* ctx = f->ctx;
  const bw_fold_spec& s = f->spec;
  // table: capacity_hint keys at a load of load_pct percent, in a whole number of segments of 2^seg_shift slots: linear
  // probing wraps inside a segment (bw_stream.cuh owns whole segments)
  const u64 load_pct = 50;
  u32 seg_shift = BW_SEG_SHIFT_DEFAULT;
  if (f->force_seg_shift >= 0) seg_shift = (u32)f->force_seg_shift;
  const u64 seg_slots = 1ULL << seg_shift;
  u64 cap = std::max<u64>(seg_slots, (std::max<u64>(s.capacity_hint, 1) * 100 + load_pct - 1) / load_pct);
  cap = (cap + seg_slots - 1) & ~(seg_slots - 1);
  if (cap > (1ULL << 31)) FAIL(f, BW_ERR_SPEC, "capacity_hint too large");
  f->t.cap = cap;
  f->t.seg_shift = seg_shift;
  f->t.seg_mask = (u32)seg_slots - 1;
  {
    // overflow pane nodes: panes a key can hold beyond its two direct slots
    const i64 per_window = f->p.panes_per_window;
    u64 expect = 32;  // wait == forever: nothing closes before EOF
    if (f->p.track_wm) expect = (u64)std::min<i64>(per_window + f->p.wait_us / f->p.pane_us + 4, 1 << 20);
    u64 want = std::max<u64>(2 * cap, std::max<u64>(s.capacity_hint, 1024) * expect) + 1024;
    // a worst-case reservation (a long wait makes `expect` huge): at most a quarter of the free device memory, so that
    // several folds fit on an 80 GB part; running out of nodes is a loud BW_ERR_CAPACITY, never a silent drop
    size_t free_b = 0, total_b = 0;
    CU(ctx, cudaMemGetInfo(&free_b, &total_b));
    want = std::min<u64>(want, (u64)(free_b / 4) / (sizeof(PaneNode) + sizeof(u64) + sizeof(u32)));
    f->t.pool_cap = (u32)std::min<u64>(want, 0x7FFFFFF0ULL);
  }
  Owner& own = f->own;
  CU(ctx, own.dev(&f->t.hot, cap + 1));
  CU(ctx, own.dev(&f->t.keys, cap + 1));
  CU(ctx, own.dev(&f->t.p1, cap + 1));
  CU(ctx, own.dev(&f->t.closed_upto, cap + 1));
  CU(ctx, own.dev(&f->t.aux, cap + 1));
  CU(ctx, own.dev(&f->t.nodes, f->t.pool_cap));
  CU(ctx, own.dev(&f->t.node_acc2, f->t.pool_cap));
  CU(ctx, own.dev(&f->t.free_stack, f->t.pool_cap));
  CU(ctx, own.dev(&f->t.dirty, cap + 2));
  CU(ctx, own.dev(&f->d_ctr, 1));
  f->t.ctr = f->d_ctr;
  CU(ctx, own.host(&f->h_ctr, 1));
  // emit buffers
  f->e.max_closed = s.max_emit_rows;
  f->e.max_late = s.max_late_rows;
  CU(ctx, own.dev(&f->e.c_key, s.max_emit_rows));
  CU(ctx, own.dev(&f->e.c_wid, s.max_emit_rows));
  CU(ctx, own.dev(&f->e.c_acc, s.max_emit_rows));
  CU(ctx, own.dev(&f->e.c_count, s.max_emit_rows));
  CU(ctx, own.dev(&f->e.c_seq, s.max_emit_rows));
  CU(ctx, own.dev(&f->e.c_epoch, s.max_emit_rows));
  CU(ctx, own.dev(&f->e.l_key, s.max_late_rows));
  CU(ctx, own.dev(&f->e.l_wid, s.max_late_rows));
  CU(ctx, own.dev(&f->e.l_val, s.max_late_rows));
  CU(ctx, own.dev(&f->e.l_ts, s.max_late_rows));
  CU(ctx, own.dev(&f->e.l_seq, s.max_late_rows));
  CU(ctx, own.dev(&f->e.l_epoch, s.max_late_rows));
  // prepass
  f->max_recv_rows = s.max_batch_rows * (u64)ctx->world;
  u64 nranges = (f->max_recv_rows + BW_RANGE_ROWS - 1) / BW_RANGE_ROWS + 1;
  CU(ctx, own.dev(&f->d_rmin, nranges));
  CU(ctx, own.dev(&f->d_rmax, nranges));
  CU(ctx, own.dev(&f->d_rbad, nranges));
  CU(ctx, own.dev(&f->d_verdict, 1));
  CU(ctx, own.dev(&f->d_span, 2));
  CU(ctx, own.host(&f->h_verdict, 64 / sizeof(u32)));
  CU(ctx, own.stream(&f->s_compute));
  CU(ctx, own.stream(&f->s_copy));
  {
    // the verdict pass gates the next fold: let its blocks be placed first whenever an SM has room
    int prio_lo = 0, prio_hi = 0;
    CU(ctx, cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    CU(ctx, own.stream(&f->s_pre, prio_hi));
  }
  CU(ctx, own.stream(&f->s_x));
  for (cudaEvent_t* e : {&f->ev_fold_done, &f->ev_xchg_done, &f->ev_pre, &f->ev_h2d})
    CU(ctx, own.event(e));
  // No persisting-L2 carve-out: a persisting window on the hot slots would leave too little normal
  // L2 for the second-pane array at window boundaries; plain LRU + evict_first input loads instead.
  int occ = 0;
  f->fold_kernel = pick_fold_kernel(f->p);
  CU(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, f->fold_kernel, BW_FOLD_THREADS, 0));
  if (occ < 1) occ = 1;
  f->fold_grid = ctx->sm_count * occ;
  // multi-GPU: leave register-file room on every SM so the next activation's partition/scatter
  // (NVLink-bound, on its own stream) can really run beside the fold instead of queueing behind it
  if (ctx->world > 1 && occ > 2) f->fold_grid = ctx->sm_count * 2;
  f->close_grid = ctx->sm_count * 8;
  {
    bw_status st = stream_alloc(f);
    if (st != BW_OK) return st;
  }
  k_init_table<<<ctx->sm_count * 8, 256, 0, f->s_compute>>>(f->t, f->p.acc_identity);
  CU(ctx, cudaGetLastError());
  f->st.kernel_launches++;
  f->st.table_capacity = cap;
  return BW_OK;
}

// one IPC-shared allocation per rank holding both receive buffers + count tables
struct XLayout {
  size_t counts_off[2], keys_off[2], vals_off[2], ts_off[2], total;
};
static XLayout xlayout(const bw_fold* f) {
  XLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t rows = (size_t)f->region_cap * f->ctx->world;
  for (int b = 0; b < 2; ++b) {
    L.counts_off[b] = take(sizeof(u64) * BW_MAX_WORLD);
    L.keys_off[b] = take(rows * 8);
    L.vals_off[b] = f->has_vals ? take(rows * (size_t)f->val_bytes) : 0;
    L.ts_off[b] = f->has_ts ? take(rows * 8) : 0;
  }
  L.total = off;
  return L;
}

static bw_status xchg_setup(bw_fold* f) {
  bw_ctx* ctx = f->ctx;
  const int W = ctx->world;
  f->region_cap = f->spec.max_batch_rows;  // worst case: every row of a source goes to one rank
  XLayout L = xlayout(f);
  f->xchg_bytes = L.total;
  Owner& own = f->own;
  CU(ctx, own.dev(&f->xchg_base, L.total));
  CU(ctx, cudaMemset(f->xchg_base, 0, L.total));
  CU(ctx, cudaFuncSetAttribute(k_part_scatter<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_PART_TILE * 24));
  u64 ntiles = (f->spec.max_batch_rows + BW_PART_TILE - 1) / BW_PART_TILE + 1;
  CU(ctx, own.dev(&f->d_tile_counts, ntiles * BW_MAX_WORLD));
  if (f->spec.exchange == BW_XCHG_P2P) {
    // every peer's receive buffer as seen from here (CUDA IPC mappings exchanged through NCCL)
    bw_status cst = coll_share_base(ctx, f->xchg_base, f->peer_base, f->s_compute);
    if (cst != BW_OK) return cst;
  } else {
    const size_t rows = (size_t)f->region_cap * W;
    CU(ctx, own.dev(&f->send_keys, rows));
    if (f->has_vals) CU(ctx, own.dev(&f->send_vals, rows * (size_t)f->val_bytes));
    if (f->has_ts) CU(ctx, own.dev(&f->send_ts, rows));
    CU(ctx, own.dev(&f->d_send_counts, BW_MAX_WORLD));
    CU(ctx, own.dev(&f->d_all_counts, (size_t)BW_MAX_WORLD * BW_MAX_WORLD));
    CU(ctx, own.host(&f->h_all_counts, (size_t)BW_MAX_WORLD * BW_MAX_WORLD));
    for (int r = 0; r < W; ++r) f->peer_base[r] = nullptr;
    f->peer_base[ctx->rank] = f->xchg_base;
  }
  return BW_OK;
}

// The environment switches, the library's only environment reads.  Tests and diagnostics use them to force a path or a
// kernel configuration that production folds reach through other shapes; they are read once, when a fold is created.
static void read_switches(bw_fold* f) {
  if (const char* e = getenv("BW_STREAM")) f->stream_mode = atoi(e) ? 1 : 0;
  if (const char* e = getenv("BW_LATE_SPLIT")) f->late_split = atoi(e) != 0;
  if (const char* e = getenv("BW_FLUSH")) f->flush_on = atoi(e) != 0;
  if (const char* e = getenv("BW_TIMER_STRIDE")) f->timer_stride = (u32)std::max(1, atoi(e));
  if (const char* e = getenv("BW_SC_STG")) f->force_stg_cap = std::max(0, std::min(16, atoi(e)));
  if (const char* e = getenv("BW_SC_EVERY")) f->force_stg_every = std::max(1, atoi(e));
  if (const char* e = getenv("BW_SC_STAGES")) f->force_nstage = std::max(2, std::min(4, atoi(e)));
  if (const char* e = getenv("BW_SEG_SHIFT")) f->force_seg_shift = std::max(10, std::min(12, atoi(e)));
}

bw_status bw_fold_create(bw_ctx* ctx, const bw_fold_spec* spec, bw_fold** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_fold_create: NULL argument");
  if (spec->struct_size != sizeof(bw_fold_spec))
    CTX_FAIL(ctx, BW_ERR_SPEC, "bw_fold_spec.struct_size %u != %zu", spec->struct_size, sizeof(bw_fold_spec));
  if (spec->reduction < 0 || spec->reduction > BW_RED_MEAN) CTX_FAIL(ctx, BW_ERR_SPEC, "bad reduction %d", spec->reduction);
  if (spec->val_dtype < 0 || spec->val_dtype > BW_VAL_F64) CTX_FAIL(ctx, BW_ERR_SPEC, "bad val_dtype %d", spec->val_dtype);
  if (spec->length_us <= 0 || spec->offset_us <= 0 || spec->offset_us > spec->length_us)
    CTX_FAIL(ctx, BW_ERR_SPEC, "need 0 < offset_us <= length_us (windowing.py:880-883)");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must be >= 0");
  if (ctx->loop && spec->exchange != BW_XCHG_P2P) CTX_FAIL(ctx, BW_ERR_SPEC, "a loopback world exchanges over peer memory only (BW_XCHG_P2P)");
  if (spec->ts_source < BW_TS_COLUMN || spec->ts_source > BW_TS_NONE) CTX_FAIL(ctx, BW_ERR_SPEC, "bad ts_source %d", spec->ts_source);
  if (spec->ts_source == BW_TS_FROM_VALUE && spec->val_dtype > BW_VAL_I64)
    CTX_FAIL(ctx, BW_ERR_SPEC, "BW_TS_FROM_VALUE needs an integer val_dtype");
  if (spec->ts_source == BW_TS_NONE && spec->wait_us != BW_WAIT_FOREVER)
    CTX_FAIL(ctx, BW_ERR_SPEC, "BW_TS_NONE (the *_final folds) needs wait_us == BW_WAIT_FOREVER: nothing closes before bw_eof");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 32) / (u64)ctx->world)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_batch_rows * world must be in [1, 2^32)");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_fold, void (*)(bw_fold*)> fp(new bw_fold(), bw_fold_destroy);  // torn down on every failure
  bw_fold* f = fp.get();
  f->ctx = ctx;
  f->spec = *spec;
  read_switches(f);
  FoldParams& p = f->p;
  p.length_us = spec->length_us;
  p.offset_us = spec->offset_us;
  p.align_us = spec->align_to_us;
  p.wait_us = spec->wait_us;
  p.pane_us = gcd_i64(spec->length_us, spec->offset_us);
  p.panes_per_offset = spec->offset_us / p.pane_us;
  p.panes_per_window = spec->length_us / p.pane_us;
  p.inv_pane = 1.0 / (double)p.pane_us;
  {
    // round-up multiplier for exact u64 division by pane_us (Granlund-Montgomery / libdivide "algorithm 1")
    const u64 D = (u64)p.pane_us;
    p.div_is_one = (D == 1);
    u32 L = 0;
    while (L < 64 && ((L == 63) ? false : ((1ULL << L) < D))) ++L;
    if ((1ULL << (L >= 64 ? 63 : L)) < D) L = 64;
    if (!p.div_is_one) {
      const unsigned __int128 one = 1;
      const unsigned __int128 num = (one << 64) * (unsigned __int128)(((L >= 64) ? (unsigned __int128)(one << 64) : (unsigned __int128)(one << L)) - D);
      p.div_magic = (u64)(num / D) + 1;
      p.div_shift = L - 1;
    } else {
      p.div_magic = 0;
      p.div_shift = 0;
    }
    // bias: multiple of pane, >= 2^59 (covers |ts - align| for every representable datetime pair)
    const i64 need = (i64)1 << 59;
    p.div_bias_q = (need + p.pane_us - 1) / p.pane_us;
    p.div_bias = p.div_bias_q * p.pane_us;
    const i64 w = p.track_wm ? p.wait_us : 0;
    p.close_back = p.length_us / p.pane_us + w / p.pane_us;
    p.wait_rem = w % p.pane_us;
  }
  p.reduction = spec->reduction;
  p.val_dtype = spec->val_dtype;
  p.ts_from_value = spec->ts_source == BW_TS_FROM_VALUE ? 1 : (spec->ts_source == BW_TS_NONE ? 2 : 0);
  p.track_wm = spec->wait_us != BW_WAIT_FOREVER;
  p.ordered = spec->ordered;
  p.need_count = spec->reduction == BW_RED_MEAN;
  // first-opened order of a key's windows == ascending id when flushes are ordered, when nothing is
  // accepted out of order (wait == 0: an accepted timestamp is never below the key's maximum), or when
  // there is a single window (the *_final folds)
  p.seq_by_id = (spec->ordered || spec->ts_source == BW_TS_NONE || spec->wait_us == 0) ? 1 : 0;
  const bool is_float = spec->val_dtype >= BW_VAL_F32, is_signed = spec->val_dtype == BW_VAL_I64;
  switch (spec->reduction) {
    case BW_RED_COUNT: p.op = BW_OP_ADD_ONE; p.acc_identity = 0; break;
    case BW_RED_SUM: p.op = is_float ? BW_OP_ADD_F64 : BW_OP_ADD_U64; p.acc_identity = 0; break;
    case BW_RED_MEAN: p.op = BW_OP_ADD_F64; p.acc_identity = 0; break;
    case BW_RED_MIN:
      p.op = (is_float || !is_signed) ? BW_OP_MIN_U64 : BW_OP_MIN_S64;
      p.acc_identity = (p.op == BW_OP_MIN_S64) ? (u64)INT64_MAX : ~0ULL;
      break;
    default:
      p.op = (is_float || !is_signed) ? BW_OP_MAX_U64 : BW_OP_MAX_S64;
      p.acc_identity = (p.op == BW_OP_MAX_S64) ? (u64)INT64_MIN : 0ULL;
      break;
  }
  f->val_bytes = spec->val_dtype == BW_VAL_F32 ? 4 : 8;
  f->has_ts = spec->ts_source == BW_TS_COLUMN;
  f->has_vals = true;  // the late stream carries the original value, even for counts
  bw_status st = fold_alloc(f);
  if (st != BW_OK) return st;
  if (ctx->world > 1) {
    st = xchg_setup(f);
    if (st != BW_OK) return st;
  }
  // emission staging is sized once: no allocation on the advance path
  const u64 n_emit = std::max<u64>(spec->max_emit_rows, spec->max_late_rows);
  CU(ctx, f->srt.reserve(f->own, n_emit, std::max<u64>(n_emit, 4096), f->s_compute));
  CU(ctx, f->ho_c.reserve(f->own, spec->max_emit_rows, std::max<u64>(spec->max_emit_rows, 4096)));
  CU(ctx, f->ho_l.reserve(f->own, spec->max_late_rows, std::max<u64>(spec->max_late_rows, 4096)));
  CU(ctx, cudaStreamSynchronize(f->s_compute));
  *out = fp.release();
  return BW_OK;
}

static bw_status stream_resolve(bw_fold* f);

void bw_fold_destroy(bw_fold* f) {
  if (!f) return;
  cudaSetDevice(f->ctx->device);
  stream_resolve(f);
  cudaDeviceSynchronize();
  for (int r = 0; r < f->ctx->world; ++r)
    if (r != f->ctx->rank && !f->ctx->loop) {
      if (f->peer_base[r] && f->spec.exchange == BW_XCHG_P2P) cudaIpcCloseMemHandle(f->peer_base[r]);
      if (f->precv_peer[r]) cudaIpcCloseMemHandle(f->precv_peer[r]);
    }
  delete f;  // f->own releases every buffer, event and stream
}

// ---------------------------------------------------------------------------
// ingest
// ---------------------------------------------------------------------------
bw_status bw_ingest_acquire(bw_fold* f, uint64_t max_rows, bw_batch* out) {
  if (!f || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (max_rows > f->spec.max_batch_rows) FAIL(f, BW_ERR_SPEC, "acquire: %llu rows > max_batch_rows", (unsigned long long)max_rows);
  CU(ctx, cudaSetDevice(ctx->device));
  const u32 nslots = f->spec.ring_slots > 0 ? (u32)f->spec.ring_slots : 3u;
  u32 pick = ~0u;
  for (u32 i = 0; i < f->slots.size(); ++i)
    if (!f->slots[i].acquired) {
      pick = i;
      break;
    }
  if (pick == ~0u) {
    if (f->slots.size() >= nslots) FAIL(f, BW_ERR_STATE, "all %u ingest slots are acquired; commit one first", nslots);
    Slot s;
    const size_t rows = f->spec.max_batch_rows;
    CU(ctx, f->own.host(&s.h_keys, rows));
    if (f->has_vals) CU(ctx, f->own.host(&s.h_vals, rows * (size_t)f->val_bytes));
    if (f->has_ts) CU(ctx, f->own.host(&s.h_ts, rows));
    f->slots.push_back(s);
    pick = (u32)f->slots.size() - 1;
  }
  Slot& s = f->slots[pick];
  s.acquired = true;
  out->keys = s.h_keys;
  out->vals = s.h_vals;
  out->ts_us = s.h_ts;
  out->capacity = f->spec.max_batch_rows;
  out->slot = pick;
  out->reserved = 0;
  return BW_OK;
}

// Time one kernel launch of activation `batch_no` on `s`: timer_begin before it, timer_end after it (`kind` and `rows` as
// in EventPair).  Every record with timing drains the stream for a few microseconds, so only every timer_stride-th
// activation is timed (env BW_TIMER_STRIDE, default 4): the averages in bw_stats are over that sample.  *ep is null when
// the launch is not timed.
static cudaError_t timer_begin(bw_fold* f, EventPair** ep, u32 batch_no, int kind, u64 rows, cudaStream_t s) {
  *ep = nullptr;
  if (f->timer_stride > 1 && batch_no % f->timer_stride != 0) return cudaSuccess;
  if (f->timers_used == f->timers.size()) {
    if (f->timers.size() >= 4096) return cudaSuccess;
    EventPair e;
    if (f->own.event(&e.a, cudaEventDefault) != cudaSuccess || f->own.event(&e.b, cudaEventDefault) != cudaSuccess) return cudaSuccess;
    f->timers.push_back(e);
  }
  *ep = &f->timers[f->timers_used++];
  (*ep)->rows = rows;
  (*ep)->kind = kind;
  return cudaEventRecord((*ep)->a, s);
}

static cudaError_t timer_end(const EventPair* ep, cudaStream_t s) { return ep ? cudaEventRecord(ep->b, s) : cudaSuccess; }

// Partition + exchange of this rank's rows; fills `bv` with the received segments.
static bw_status exchange(bw_fold* f, const u64* d_keys, const void* d_vals, const i64* d_ts, u64 rows, BatchView* bv) {
  bw_ctx* ctx = f->ctx;
  const int W = ctx->world, R = ctx->rank;
  // Partition + exchange run on their own stream so that the scatter of activation b+1 (NVLink-bound)
  // overlaps the fold of activation b.  The producer of the input columns is ordered before it through
  // cols_ready; the barrier waits for this rank's fold of the previous activation, which is what makes
  // the double-buffered receive regions safe to overwrite two activations later.
  cudaStream_t s = f->s_x;
  if (f->cols_ready) CU(ctx, cudaStreamWaitEvent(s, f->cols_ready, 0));
  const int buf = f->xbuf;
  f->xbuf ^= 1;
  XLayout L = xlayout(f);
  PartIn in;
  in.keys = d_keys;
  in.vals = d_vals;
  in.ts = f->has_ts ? d_ts : nullptr;
  in.n = rows;
  in.val_bytes = d_vals ? f->val_bytes : 0;
  in.world = W;
  PartOut po;
  memset(&po, 0, sizeof po);
  po.region_cap = f->region_cap;
  const bool p2p = f->spec.exchange == BW_XCHG_P2P;
  const bool hv = d_vals != nullptr;  // counts may come without a value column
  for (int d = 0; d < W; ++d) {
    if (p2p) {
      char* base = (char*)f->peer_base[d];
      po.keys[d] = (u64*)(base + L.keys_off[buf]) + (size_t)R * f->region_cap;
      po.vals[d] = hv ? (void*)(base + L.vals_off[buf] + (size_t)R * f->region_cap * f->val_bytes) : nullptr;
      po.ts[d] = f->has_ts ? (i64*)(base + L.ts_off[buf]) + (size_t)R * f->region_cap : nullptr;
      po.counts[d] = (u64*)(base + L.counts_off[buf]) + R;
    } else {
      po.keys[d] = f->send_keys + (size_t)d * f->region_cap;
      po.vals[d] = hv ? (void*)((char*)f->send_vals + (size_t)d * f->region_cap * f->val_bytes) : nullptr;
      po.ts[d] = f->has_ts ? f->send_ts + (size_t)d * f->region_cap : nullptr;
      po.counts[d] = f->d_send_counts + d;
    }
  }
  const u64 ntiles = (rows + BW_PART_TILE - 1) / BW_PART_TILE;
  int grid = (int)std::min<u64>(std::max<u64>(ntiles, 1), (u64)ctx->sm_count * 8);
  k_part_hist<<<grid, BW_PART_THREADS, 0, s>>>(in, f->d_tile_counts);
  k_part_scan<<<W, 1024, 0, s>>>(rows, W, f->d_tile_counts, po, f->d_ctr);
  const size_t stage_bytes = (size_t)BW_PART_TILE * (8 + (size_t)in.val_bytes + (in.ts ? 8 : 0));
  k_part_scatter<false><<<grid, BW_PART_THREADS, stage_bytes, s>>>(in, f->d_tile_counts, po, PartSide{});
  CU(ctx, cudaGetLastError());
  f->st.kernel_launches += 3;
  char* mine = (char*)f->xchg_base;
  u64* my_counts = (u64*)(mine + L.counts_off[buf]);
  if (f->fold_recorded) CU(ctx, cudaStreamWaitEvent(s, f->ev_fold_done, 0));
  if (p2p) {
    // every rank's stores are complete once it enters this collective (stream
    // order); its completion here means all peers have entered it.
    {
      bw_status cst = coll_barrier(ctx, f->d_verdict, s);
      if (cst != BW_OK) return cst;
    }
  } else {
    NC(ctx, ncclAllGather(f->d_send_counts, f->d_all_counts, BW_MAX_WORLD, ncclUint64, ctx->comm, s));
    CU(ctx, cudaMemcpyAsync(f->h_all_counts, f->d_all_counts, sizeof(u64) * BW_MAX_WORLD * W, cudaMemcpyDeviceToHost, s));
    CU(ctx, cudaStreamSynchronize(s));
    u64 recv_counts[BW_MAX_WORLD];
    NC(ctx, ncclGroupStart());
    for (int r = 0; r < W; ++r) {
      const u64 nsend = f->h_all_counts[(size_t)R * BW_MAX_WORLD + r];
      const u64 nrecv = f->h_all_counts[(size_t)r * BW_MAX_WORLD + R];
      recv_counts[r] = nrecv;
      u64* rk = (u64*)(mine + L.keys_off[buf]) + (size_t)r * f->region_cap;
      NC(ctx, ncclSend(f->send_keys + (size_t)r * f->region_cap, nsend, ncclUint64, r, ctx->comm, s));
      NC(ctx, ncclRecv(rk, nrecv, ncclUint64, r, ctx->comm, s));
      if (hv) {
        char* rv = mine + L.vals_off[buf] + (size_t)r * f->region_cap * f->val_bytes;
        NC(ctx, ncclSend((char*)f->send_vals + (size_t)r * f->region_cap * f->val_bytes, nsend * f->val_bytes, ncclChar, r,
                         ctx->comm, s));
        NC(ctx, ncclRecv(rv, nrecv * f->val_bytes, ncclChar, r, ctx->comm, s));
      }
      if (f->has_ts) {
        i64* rt = (i64*)(mine + L.ts_off[buf]) + (size_t)r * f->region_cap;
        NC(ctx, ncclSend(f->send_ts + (size_t)r * f->region_cap, nsend, ncclInt64, r, ctx->comm, s));
        NC(ctx, ncclRecv(rt, nrecv, ncclInt64, r, ctx->comm, s));
      }
    }
    NC(ctx, ncclGroupEnd());
    CU(ctx, cudaMemcpyAsync(my_counts, recv_counts, sizeof(u64) * W, cudaMemcpyHostToDevice, s));
    // recv_counts is a stack array: make the copy complete before returning
    CU(ctx, cudaStreamSynchronize(s));
  }
  memset(bv, 0, sizeof *bv);
  bv->nseg = W;
  bv->counts_on_device = 1;
  bv->d_counts = my_counts;
  bv->max_rows = f->max_recv_rows;
  for (int r = 0; r < W; ++r) {
    bv->keys[r] = (const u64*)(mine + L.keys_off[buf]) + (size_t)r * f->region_cap;
    bv->vals[r] = hv ? (const void*)(mine + L.vals_off[buf] + (size_t)r * f->region_cap * f->val_bytes) : nullptr;
    bv->ts[r] = f->has_ts ? (const i64*)(mine + L.ts_off[buf]) + (size_t)r * f->region_cap : nullptr;
  }
  return BW_OK;
}

// K4 for the keys the fold marked, then the end-of-activation resets
static bw_status close_stage(bw_fold* f, u64 ord, u32 batch_no, StreamVerdict* sv) {
  bw_ctx* ctx = f->ctx;
  k_close_dirty<<<f->close_grid, 256, 0, f->s_compute>>>(f->t, f->p, f->e, ord, batch_no);
  k_stream_reset<<<1, 1, 0, f->s_compute>>>(f->t, sv);
  CU(ctx, cudaGetLastError());
  f->st.kernel_launches += 2;
  return BW_OK;
}

// The direct fold kernel over a clean activation, in sub-ranges when it spans several panes.
static bw_status direct_fold(bw_fold* f, const BatchView& bv, u64 known, u32 batch_no, u64 ord, i64 tmin, i64 tmax) {
  bw_ctx* ctx = f->ctx;
  const u64 tile = (u64)BW_FOLD_THREADS * BW_FOLD_UNROLL;
  // Fold + close in sub-ranges of the activation (by arrival index, resolved on the device so
  // that it also works on exchanged rows whose counts the host never sees).  Windows a key has
  // left are closed -- and its newest pane promoted into the hot slot -- between sub-ranges, so
  // an activation that spans several windows (8 ranks x 2^24 rows of C1 = 134 s of event time
  // per activation) keeps hitting the two direct panes instead of the overflow list.  Rows are
  // identical: a pane closed early would also close at the end (the watermark only grows, and
  // the pane holding max_ts never closes).  One sub-range per pane of event-time span, for
  // in-order streams; activations inside one pane (C1 on one GPU) are not split.
  u32 n_sub = 1;
  if (f->p.track_wm && tmax > tmin) {
    const u64 panes = (u64)(tmax - tmin) / (u64)f->p.pane_us + (((u64)(tmax - tmin) % (u64)f->p.pane_us) ? 1 : 0);
    n_sub = (u32)std::min<u64>(panes, 8);
    n_sub = (u32)std::min<u64>(n_sub, std::max<u64>(known >> 20, 1));  // keep sub-ranges >= 2^20 rows
  }
  for (u32 i = 0; i < n_sub; ++i) {
    const u64 n_hi = (known * (i + 1ULL)) / n_sub, n_lo = (known * (u64)i) / n_sub;
    EventPair* ep;
    CU(ctx, timer_begin(f, &ep, batch_no, 0, (ctx->world > 1) ? 0 : (n_hi - n_lo), f->s_compute));
    int grid = (int)std::min<u64>((n_hi - n_lo + tile - 1) / tile + 1, (u64)f->fold_grid);
    f->fold_kernel<<<grid, BW_FOLD_THREADS, 0, f->s_compute>>>(bv, f->t, f->p, batch_no, i, n_sub);
    CU(ctx, cudaGetLastError());
    CU(ctx, timer_end(ep, f->s_compute));
    f->st.kernel_launches++;
    f->st.fold_launches++;
    if (i + 1 < n_sub) {
      k_close_dirty<<<f->close_grid, 256, 0, f->s_compute>>>(f->t, f->p, f->e, ord, batch_no);
      k_reset_dirty<<<1, 1, 0, f->s_compute>>>(f->t);
      f->st.kernel_launches += 2;
    }
  }
  return BW_OK;
}

// ---- streaming path (bw_stream.cuh): queue scatter + verdict now, the fold stage one activation later ----
static bool stream_usable(const bw_fold* f, const u64* d_keys, const void* d_vals, const i64* d_ts, u64 rows) {
  if (!f->stream_ok || rows == 0 || rows > f->spec.max_batch_rows) return false;
  // 128-bit loads of column pairs
  if (((uintptr_t)d_keys & 15) || ((uintptr_t)d_vals & 15) || ((uintptr_t)d_ts & 15)) return false;
  if (f->p.ts_from_value == 1 && !d_vals) return false;
  if (f->sb.val_bytes && !d_vals) return false;
  return true;
}

static bw_status stream_front(bw_fold* f, const u64* d_keys, const void* d_vals, const i64* d_ts, u64 rows, u32 batch_no, int side,
                              const u32* late_bits = nullptr, i64 ts0 = 0) {
  bw_ctx* ctx = f->ctx;
  const StreamBufs& sb = f->sb;
  cudaStream_t s = f->s_compute;
  ScatterArgs A;
  memset(&A, 0, sizeof A);
  A.keys = d_keys;
  A.vals = d_vals;
  A.ts = f->has_ts ? d_ts : nullptr;
  A.n = rows;
  A.out = sb.side[side];
  A.nb = sb.nb;
  A.nlanes = sb.nlanes;
  A.lane_cap = sb.lane_cap;
  A.spill_cap = sb.spill_cap;
  A.tile_min = sb.tile_min + (size_t)side * sb.tiles_cap;
  A.tile_max = sb.tile_max + (size_t)side * sb.tiles_cap;
  A.tile_bad = sb.tile_bad + (size_t)side * sb.tiles_cap;
  A.chunk_max = sb.chunk_max + (size_t)side * sb.tiles_cap * BW_SC_WARPS;
  A.late_bits = late_bits;  // second run over an activation with late rows: they are left out
  A.ts0_set = late_bits ? 1u : 0u;
  A.ts0 = ts0;
  A.cap = f->t.cap;
  A.seg_shift = f->t.seg_shift;
  A.nstage = (u32)f->scatter_nstage;
  A.rec_idx = f->p.seq_by_id ? 0u : 1u;
  A.stg_cap = f->scatter_stg_cap;
  A.stg_every = f->scatter_stg_every;
  A.ovf_cap = f->scatter_ovf_cap;
  A.batch_no = batch_no;
  A.world = (u32)ctx->world;
  A.nb_local = f->nb_local;
  const bool multi = ctx->world > 1;
  // multi-GPU: every rank goes through here for every activation (the verdicts are gathered collectively); a rank
  // whose columns the scatter cannot read (no rows, unaligned) sends no rows / asks everyone for the legacy path
  const bool usable = stream_usable(f, d_keys, d_vals, d_ts, rows);
  VerdictGather* vg = multi ? f->d_vg_local + side : nullptr;
  const u64 T = BW_SC_TILE;
  const u64 ntiles = usable ? (rows + T - 1) / T : 0;
  const int grid = (int)std::min<u64>(ntiles, (u64)std::min<u32>((u32)f->scatter_grid, sb.nlanes));
  f->last_scatter_grid = (u32)grid;
  if (multi && !usable && rows) CU(ctx, cudaMemsetAsync(&sb.side[side].sv->flags, 0xFF, sizeof(u32), s));  // every flag: legacy path
  EventPair* ep;
  CU(ctx, timer_begin(f, &ep, batch_no, 1, rows, s));
  if (grid) f->scatter_kernel<<<grid, BW_SC_THREADS, f->scatter_smem, s>>>(A, f->p);
  CU(ctx, timer_end(ep, s));  // (the scatter kernel alone: the one-block verdict is timed apart)
  CU(ctx, timer_begin(f, &ep, batch_no, 2, 0, s));
  if (f->p.ts_from_value == 2) k_verdict_none<<<1, 1, 0, s>>>(f->p, f->d_ctr, sb.side[side].sv, vg, rows);
  else
    k_verdict<<<1, 1024, 0, s>>>(A.tile_min, A.tile_max, A.tile_bad, (u32)ntiles, f->p, f->d_ctr, sb.side[side].sv,
                                 f->has_ts ? d_ts : nullptr, (const u64*)d_vals, vg);
  CU(ctx, cudaGetLastError());
  CU(ctx, timer_end(ep, s));
  f->st.kernel_launches += 2;
  CU(ctx, cudaMemcpyAsync(&f->h_sv[side], sb.side[side].sv, sizeof(StreamVerdict), cudaMemcpyDeviceToHost, s));
  if (multi) f->vg_pending[side] = true;  // gathered by the next collective on the stream (gather_verdict)
  CU(ctx, cudaEventRecord(f->ev_sv[side], s));
  return BW_OK;
}

static bw_status slow_path(bw_fold* f, const BatchView& bv, u64 total, u64 epoch_ord, u32 batch_no);

// The caller's columns of activation d as one segment.
static BatchView one_segment(const bw_fold* f, const Deferred& d) {
  BatchView bv;
  memset(&bv, 0, sizeof bv);
  bv.nseg = 1;
  bv.keys[0] = d.d_keys;
  bv.vals[0] = d.d_vals;
  bv.ts[0] = f->has_ts ? d.d_ts : nullptr;
  bv.h_counts[0] = d.rows;
  bv.max_rows = d.rows;
  return bv;
}

// The segment-fold arguments of streamed activation d that every mode shares.  The span (ts0, q_lo, npass) and the
// multi-GPU fields are the caller's.
static SegArgs seg_args(const bw_fold* f, const Deferred& d) {
  const StreamBufs& sb = f->sb;
  SegArgs A;
  memset(&A, 0, sizeof A);
  A.in = sb.side[d.side];
  A.nb = sb.nb;
  A.nlanes = sb.nlanes;
  A.lane_cap = sb.lane_cap;
  A.nlanes_used = d.lanes;
  A.spill_cap = sb.spill_cap;
  A.val_bytes = sb.val_bytes;
  A.seg_shift = f->t.seg_shift;
  A.batch_no = d.batch_no;
  A.epoch = d.ord;
  A.parts = f->segfold_parts;
  return A;
}

// The lateness pass over activation d's rows on this rank (bw_prepass.cuh); on world > 1 behind the partition + exchange
// of the raw rows, which point *bv at the received segments.  *clean: no row can be late, and [*tmin, *tmax] is the
// span of its event times (0 when the fold keeps no watermark).
static bw_status prepass(bw_fold* f, const Deferred& d, BatchView* bv, bool* clean, i64* tmin, i64* tmax) {
  bw_ctx* ctx = f->ctx;
  u64 max_total = d.rows;
  cudaStream_t pre_stream = f->s_pre;
  if (ctx->world > 1) {
    bw_status st = exchange(f, d.d_keys, d.d_vals, d.d_ts, d.rows, bv);
    if (st != BW_OK) return st;
    max_total = f->max_recv_rows;
    pre_stream = f->s_x;  // the verdict is computed right behind the exchange, beside the previous fold
  }
  *clean = true;
  *tmin = *tmax = 0;
  if (f->p.track_wm && max_total > 0) {
    if (ctx->world == 1 && f->cols_ready) CU(ctx, cudaStreamWaitEvent(pre_stream, f->cols_ready, 0));
    const u64 nranges = (max_total + BW_RANGE_ROWS - 1) / BW_RANGE_ROWS;
    // one warp per 2048-row range; cap at 64 warps per SM in total (the block size is small so that a block fits beside the fold)
    int grid = (int)std::min<u64>((nranges * 32 + BW_PRE_THREADS - 1) / BW_PRE_THREADS, (u64)ctx->sm_count * (2048 / BW_PRE_THREADS));
    if (grid < 1) grid = 1;
    k_prepass_ranges<<<grid, BW_PRE_THREADS, 0, pre_stream>>>(*bv, f->p, f->d_rmin, f->d_rmax, f->d_rbad);
    k_prepass_scan<<<1, 1024, 0, pre_stream>>>(*bv, f->p, f->d_rmin, f->d_rmax, f->d_rbad, f->d_ctr, f->d_verdict, f->d_span);
    CU(ctx, cudaGetLastError());
    f->st.kernel_launches += 2;
    CU(ctx, cudaMemcpyAsync(f->h_verdict, f->d_verdict, sizeof(u32), cudaMemcpyDeviceToHost, pre_stream));
    CU(ctx, cudaMemcpyAsync(f->h_verdict + 4, f->d_span, 2 * sizeof(i64), cudaMemcpyDeviceToHost, pre_stream));
    CU(ctx, cudaEventRecord(f->ev_pre, pre_stream));
    CU(ctx, cudaEventSynchronize(f->ev_pre));
    *clean = (*f->h_verdict != 0);
    *tmin = ((const i64*)(f->h_verdict + 4))[0];
    *tmax = ((const i64*)(f->h_verdict + 4))[1];
    if (pre_stream != f->s_compute) CU(ctx, cudaStreamWaitEvent(f->s_compute, f->ev_pre, 0));
  }
  if (ctx->world > 1) {  // the fold may start once the exchange (and the verdict pass behind it) is done
    CU(ctx, cudaEventRecord(f->ev_xchg_done, f->s_x));
    CU(ctx, cudaStreamWaitEvent(f->s_compute, f->ev_xchg_done, 0));
  }
  return BW_OK;
}

// One collective per activation: the all-gather that brings every rank's verdict of the activation just scattered is
// also the barrier behind the previous activation's combine (a rank enters it after its peer stores, in stream order).
static bw_status gather_verdict(bw_fold* f, int side) {
  bw_ctx* ctx = f->ctx;
  cudaStream_t s = f->s_compute;
  const int W = ctx->world;
  VerdictGather* all = f->d_vg_all + (size_t)side * W;
  {
    bw_status cst = coll_allgather(ctx, f->d_vg_local + side, all, sizeof(VerdictGather), s);
    if (cst != BW_OK) return cst;
  }
  CU(ctx, cudaMemcpyAsync(f->h_vg + (size_t)side * W, all, sizeof(VerdictGather) * W, cudaMemcpyDeviceToHost, s));
  if (!f->ev_vg[side]) CU(ctx, f->own.event(&f->ev_vg[side]));
  CU(ctx, cudaEventRecord(f->ev_vg[side], s));
  f->vg_pending[side] = false;
  return BW_OK;
}

// World > 1: combine -> partials over NVLink -> barrier -> merge for streamed activation d, when the gathered verdicts
// of every rank allow it (*folded).  Every rank has the same gathered verdicts, so every rank takes the same branch and
// the collectives line up.  *running: the maximum event time over all ranks after d.
static bw_status combine_merge(bw_fold* f, const Deferred& d, bool* folded, i64* running) {
  bw_ctx* ctx = f->ctx;
  const StreamBufs& sb = f->sb;
  const FoldParams& p = f->p;
  cudaStream_t s = f->s_compute;
  const int W = ctx->world, R = ctx->rank;
  const StreamVerdict sv = f->h_sv[d.side];
  *folded = false;
  f->st.scatter_spill_rows += sv.n_spill;
  // this activation's verdicts: gathered by the previous activation's exchange barrier, else (first activation, or
  // after a flush) by a collective of their own
  if (f->vg_pending[d.side]) {
    bw_status gst = gather_verdict(f, d.side);
    if (gst != BW_OK) return gst;
  }
  CU(ctx, cudaEventSynchronize(f->ev_vg[d.side]));
  const int next_side = d.side ^ 1;  // the activation scattered after this one (if any) waits for its gather
  const VerdictGather* vg = f->h_vg + (size_t)d.side * W;
  // chain the ranks' slices in source order: the arrival order at every destination (bw_prepass.cuh's rule)
  i64 gmin = INT64_MAX, gmax = INT64_MIN;
  *running = f->h_gmax;
  bool bad = false, unfit = false;
  for (int r = 0; r < W; ++r) {
    if (vg[r].flags || vg[r].n_spill) unfit = true;  // a row some scatter set aside belongs to another rank's table
    if (vg[r].tmax < vg[r].tmin) continue;            // no rows on that rank
    if (vg[r].bad || vg[r].tmin < bw_sub_sat(*running, p.wait_us)) bad = true;
    *running = std::max(*running, vg[r].tmax);
    gmin = std::min(gmin, vg[r].tmin);
    gmax = std::max(gmax, vg[r].tmax);
    // the combine folds a rank's slice in one pass: two panes
    if (bw_floordiv(vg[r].tmax - p.align_us, p.pane_us) - bw_floordiv(vg[r].tmin - p.align_us, p.pane_us) > 1) unfit = true;
  }
  const bool any_rows = gmax >= gmin;
  const bool clean = !p.track_wm || !bad;
  i64 q_lo = 0, q_hi = 0;
  if (any_rows) {
    q_lo = bw_floordiv(gmin - p.align_us, p.pane_us);
    q_hi = bw_floordiv(gmax - p.align_us, p.pane_us);
    if ((u64)(gmax - gmin) >= 0x7FFFFFF0ULL || q_hi - q_lo >= 2 * 64) unfit = true;
  }
  f->h_gmax = *running;
  k_set_gmax<<<1, 1, 0, s>>>(f->d_ctr, *running);  // (the legacy path's lateness pass chains from the same maximum)
  f->st.kernel_launches++;
  if (!clean || unfit) {
    if (f->vg_pending[next_side]) return gather_verdict(f, next_side);
    return BW_OK;
  }
  f->st.rows_received += d.rows;  // (this rank's share of the rows arrives as partials)
  SegArgs A = seg_args(f, d);
  A.world = (u32)W;
  A.rank = (u32)R;
  A.nb_local = f->nb_local;
  A.part_cap = f->part_cap;
  for (int r = 0; r < W; ++r) {
    char* base = (char*)f->precv_peer[r];
    A.pcnt_out[r] = (u32*)(base + f->precv_cnt_off[d.side]) + (size_t)R * f->nb_local;
    A.pout[r] = (Partial*)(base + f->precv_rec_off[d.side]) + (size_t)R * f->nb_local * f->part_cap;
  }
  A.pcnt_in = (const u32*)((char*)f->precv_base + f->precv_cnt_off[d.side]);
  A.pin = (const Partial*)((char*)f->precv_base + f->precv_rec_off[d.side]);
  EventPair* ep;
  CU(ctx, timer_begin(f, &ep, d.batch_no, 0, d.rows, s));
  // combine this rank's slice (one pass over its own two panes) and store the partials in their owners' regions
  A.ts0 = sv.ts0;
  A.q_lo = (sv.tmax >= sv.tmin) ? bw_floordiv(sv.tmin - p.align_us, p.pane_us) : 0;
  A.npass = 1;
  f->combine_kernel<<<(int)std::min<u32>(sb.nb, (u32)f->combine_grid), BW_SF_THREADS, f->segfold_smem, s>>>(A, f->t, f->p, f->e);
  CU(ctx, cudaGetLastError());
  // every rank's partials are in place once every rank has entered this collective -- which also carries the verdicts
  // of the activation scattered after this one
  if (f->vg_pending[next_side]) {
    bw_status gst = gather_verdict(f, next_side);
    if (gst != BW_OK) return gst;
  } else {
    bw_status cst = coll_barrier(ctx, f->d_barrier_word, s);
    if (cst != BW_OK) return cst;
  }
  // merge what every source left for this rank's segments, in source order, over the activation's whole span
  A.nb = f->nb_local;
  A.ts0 = any_rows ? gmin : p.align_us;
  A.q_lo = q_lo;
  A.npass = (u32)((q_hi - q_lo) / 2 + 1);
  f->merge_kernel<<<(int)std::min<u32>(f->nb_local, (u32)f->merge_grid), BW_SF_THREADS, f->segfold_smem, s>>>(A, f->t, f->p, f->e);
  CU(ctx, cudaGetLastError());
  CU(ctx, timer_end(ep, s));
  k_spill<<<ctx->sm_count, 256, 0, s>>>(f->t, f->p, sb.side[d.side].spill, sb.side[d.side].sv, sb.spill_cap, d.batch_no, 0u, 0xFFFFFFFFu);
  f->st.kernel_launches += 3;
  f->st.fold_launches++;
  f->st.combined_folds++;
  *folded = true;
  return BW_OK;
}

// An activation the verdict could not prove clean (one GPU): find its late rows without sorting it (bw_late.cuh), then
// scatter it again without them.  *ok: *sv is now the verdict of the rows that are left -- none of them late, so the
// streaming fold is exact for them -- and the late rows wait in f->late for k_late_emit.  Not ok (more suspects than
// the table takes, or the second scatter raised a flag): nothing has been folded or emitted, take the sort path.
static bw_status late_split(bw_fold* f, const Deferred& d, const BatchView& bv, StreamVerdict* sv, bool* ok) {
  bw_ctx* ctx = f->ctx;
  const StreamBufs& sb = f->sb;
  cudaStream_t s = f->s_compute;
  *ok = false;
  LateBufs& L = f->late;
  if (!f->late_ready) {
    const u64 maxr = f->spec.max_batch_rows;
    L.cap = (u32)std::max<u64>(1024, maxr / 16);
    u32 M = 2048;
    while (M < 2 * L.cap) M <<= 1;
    L.m_mask = M - 1;
    u32 kb = 1u << 16;
    while (kb < 16 * L.cap && kb < (1u << 27)) kb <<= 1;
    L.kb_mask = kb - 1;
    Owner& own = f->own;
    CU(ctx, own.dev(&L.key_bits, kb / 32));
    CU(ctx, own.dev(&L.late_bits, maxr / 32 + 2));
    CU(ctx, own.dev(&L.ent, M));
    CU(ctx, cudaMemsetAsync(L.ent, 0, (size_t)M * sizeof(LateEnt), s));  // generation 0: every entry free, once
    CU(ctx, own.dev(&L.counters, 2));
    CU(ctx, own.dev(&L.s_key, L.cap));
    CU(ctx, own.dev(&L.s_ts, L.cap));
    CU(ctx, own.dev(&L.s_idx, L.cap));
    CU(ctx, own.dev(&L.s_slot, L.cap));
    CU(ctx, own.dev(&L.gpre, sb.tiles_cap));
    CU(ctx, own.dev(&f->late_chunk_pre, (size_t)sb.tiles_cap * BW_SC_WARPS));
    CU(ctx, own.host(&f->h_late_ctr, 2));
    f->late_ready = true;
  }
  const u64 rows = d.rows;
  const u32 ntiles = (u32)((rows + BW_SC_TILE - 1) / BW_SC_TILE);
  CU(ctx, cudaMemsetAsync(L.key_bits, 0, ((size_t)L.kb_mask + 1) / 8, s));
  CU(ctx, cudaMemsetAsync(L.late_bits, 0, (rows / 32 + 2) * sizeof(u32), s));
  L.gen = d.batch_no + 1u;  // (batch numbers of a fold never repeat)
  CU(ctx, cudaMemsetAsync(L.counters, 0, 2 * sizeof(u32), s));
  const size_t toff = (size_t)d.side * sb.tiles_cap;
  const int wide = ctx->sm_count * 8;
  k_late_gpre<<<1, 1024, 0, s>>>(sb.tile_max + toff, ntiles, sv->gprev, L.gpre);
  k_late_chunkpre<<<(int)std::min<u32>((ntiles + 7u) / 8u, (u32)wide), 256, 0, s>>>(sb.chunk_max + toff * BW_SC_WARPS, L.gpre, ntiles, f->late_chunk_pre);
  k_late_suspect<<<wide, 256, 0, s>>>(bv, f->p, rows, f->late_chunk_pre, L);
  k_late_build<<<wide, 256, 0, s>>>(L);
  k_late_prefmax<<<wide, 256, 0, s>>>(bv, f->p, rows, L);
  k_late_classify<<<wide, 256, 0, s>>>(f->t, f->p, L);
  k_stream_reset<<<1, 1, 0, s>>>(f->t, sb.side[d.side].sv);  // what the first scatter set aside / flagged is void
  CU(ctx, cudaGetLastError());
  f->st.kernel_launches += 7;
  CU(ctx, cudaMemcpyAsync(f->h_late_ctr, L.counters, 2 * sizeof(u32), cudaMemcpyDeviceToHost, s));
  // base of the records' 32-bit relative timestamps: row 0 may be a late row from far back, so count from the
  // activation's newest timestamp instead
  i64 ts0 = sv->tmin;
  if (sv->tmax - (i64)0x7FFFFFF0 > ts0) ts0 = sv->tmax - (i64)0x7FFFFFF0;
  bw_status st = stream_front(f, d.d_keys, d.d_vals, d.d_ts, rows, d.batch_no, d.side, L.late_bits, ts0);
  if (st != BW_OK) return st;
  CU(ctx, cudaEventSynchronize(f->ev_sv[d.side]));
  if (f->h_late_ctr[0] > L.cap || f->h_late_ctr[1]) return BW_OK;
  const StreamVerdict sv2 = f->h_sv[d.side];
  if (sv2.flags) return BW_OK;
  *sv = sv2;
  sv->clean = 1u;
  sv->ts0 = ts0;
  *ok = true;
  return BW_OK;
}

// One GPU: the segment fold of streamed activation d (bv: its columns), when its verdict allows (*folded) -- after the
// late-row split of an activation the verdict could not prove clean.  *sv: the verdict the fold stage goes by.
static bw_status segment_fold(bw_fold* f, const Deferred& d, const BatchView& bv, StreamVerdict* sv, bool* folded) {
  bw_ctx* ctx = f->ctx;
  const StreamBufs& sb = f->sb;
  const FoldParams& p = f->p;
  cudaStream_t s = f->s_compute;
  *sv = f->h_sv[d.side];
  bool split = false;
  if (!sv->clean && p.track_wm && f->late_split) {
    bw_status lst = late_split(f, d, bv, sv, &split);
    if (lst != BW_OK) return lst;
  }
  f->st.scatter_spill_rows += sv->n_spill;
  i64 q_lo = 0, q_hi = 0;
  if (sv->tmax >= sv->tmin) {
    q_lo = bw_floordiv(sv->tmin - p.align_us, p.pane_us);
    q_hi = bw_floordiv(sv->tmax - p.align_us, p.pane_us);
  }
  *folded = sv->clean && !sv->flags && (q_hi - q_lo) < 2 * 64;
  if (!*folded) {
    // (the scatter output of this activation is simply not read)
    if (split) *sv = f->h_sv[d.side], sv->clean = 0u;  // (split, but too many panes for the segment fold: the sort path; nothing was emitted)
    return BW_OK;
  }
  SegArgs A = seg_args(f, d);
  A.ts0 = sv->ts0;
  A.q_lo = q_lo;
  A.npass = (u32)((q_hi - q_lo) / 2 + 1);
  EventPair* ep;
  CU(ctx, timer_begin(f, &ep, d.batch_no, 0, d.rows, s));
  if (split) {
    k_late_emit<<<ctx->sm_count * 4, 256, 0, s>>>(bv, f->t, f->p, f->e, f->late, d.batch_no, d.ord);
    f->st.kernel_launches++;
    f->st.split_batches++;
  }
  const u32 n_pre = std::min<u32>(sv->n_spill, sb.spill_cap);  // rows the scatter set aside: fold them first
  if (n_pre) {
    k_spill<<<(int)std::min<u32>((n_pre + 255) / 256, (u32)ctx->sm_count * 4), 256, 0, s>>>(f->t, f->p, sb.side[d.side].spill, sb.side[d.side].sv,
                                                                                           sb.spill_cap, d.batch_no, 0u, n_pre);
    f->st.kernel_launches++;
  }
  const int grid = (int)std::min<u32>(sb.nb, (u32)f->segfold_grid);
  f->segfold_kernel<<<grid, BW_SF_THREADS, f->segfold_smem, s>>>(A, f->t, f->p, f->e);
  CU(ctx, cudaGetLastError());
  CU(ctx, timer_end(ep, s));
  k_spill<<<ctx->sm_count, 256, 0, s>>>(f->t, f->p, sb.side[d.side].spill, sb.side[d.side].sv, sb.spill_cap, d.batch_no, n_pre, 0xFFFFFFFFu);
  f->st.kernel_launches += 2;
  f->st.fold_launches++;
  f->st.combined_folds++;
  return BW_OK;
}

// The fold stage of activation d, whose columns are on the device: `streamed` when its scatter + verdict are queued
// (the deferred activation).  A streamed activation takes the segment fold (one GPU) or combine + merge (world > 1) when
// its verdict allows.  Otherwise the direct kernel folds it when it is clean, else the sort path; whether it is clean is
// the streamed verdict on one GPU, else the lateness pass over the caller's columns or, on world > 1, over the rows
// the exchange brought.  Every path ends in the same tail: close, mark the rows (one GPU) or record the fold's end (world
// > 1), release the staging buffer.
static bw_status fold_stage(bw_fold* f, const Deferred& d, bool streamed) {
  bw_ctx* ctx = f->ctx;
  const bool multi = ctx->world > 1;
  cudaStream_t s = f->s_compute;
  StreamVerdict* dsv = f->sb.side[d.side].sv;  // (streamed) the scatter's verdict on the device
  BatchView bv = one_segment(f, d);
  StreamVerdict sv{};
  bool folded = false;
  i64 running = 0;
  bw_status st = BW_OK;
  if (streamed) {
    st = multi ? combine_merge(f, d, &folded, &running) : segment_fold(f, d, bv, &sv, &folded);
    if (st != BW_OK) return st;
  }
  const bool prepassed = !folded && (multi || !streamed);
  bool clean = sv.clean;
  i64 tmin = sv.tmin, tmax = sv.tmax;
  if (prepassed && (st = prepass(f, d, &bv, &clean, &tmin, &tmax)) != BW_OK) return st;
  const bool any = multi || d.rows > 0;  // (on world > 1 the exchange may bring rows to a rank that has none)
  if (!folded && any) {
    if (clean) {
      st = direct_fold(f, bv, multi ? f->max_recv_rows : d.rows, d.batch_no, d.ord, tmin, tmax);
    } else {
      u64 total = d.rows;
      if (multi) {
        u64 hc[BW_MAX_WORLD];
        CU(ctx, cudaMemcpyAsync(hc, bv.d_counts, sizeof(u64) * ctx->world, cudaMemcpyDeviceToHost, s));
        CU(ctx, cudaStreamSynchronize(s));
        total = 0;
        for (int r = 0; r < ctx->world; ++r) total += hc[r];
      }
      st = slow_path(f, bv, total, d.ord, d.batch_no);
      f->st.slow_batches++;
    }
    if (st != BW_OK) return st;
  }
  // the scatter's verdict is reset with the close, unless the rows went through the lateness pass instead
  if (any && (st = close_stage(f, d.ord, d.batch_no, streamed && !prepassed ? dsv : nullptr)) != BW_OK) return st;
  if (streamed && prepassed) {  // (world > 1) the scatter's verdict, and the chain's maximum the lateness pass moved
    k_stream_reset<<<1, 1, 0, s>>>(f->t, dsv);
    k_set_gmax<<<1, 1, 0, s>>>(f->d_ctr, running);
  }
  if (multi) {
    CU(ctx, cudaEventRecord(f->ev_fold_done, s));
    f->fold_recorded = true;
  } else if ((st = mark_rows(f, d.ord)) != BW_OK) {
    return st;
  }
  if (d.stage) {
    CU(ctx, cudaEventRecord(d.stage->consumed, s));
    d.stage->used = true;
  }
  return BW_OK;
}

static bw_status stream_resolve(bw_fold* f) {
  Deferred d = f->dq;
  if (!d.valid) return BW_OK;
  f->dq.valid = false;
  CU(f->ctx, cudaEventSynchronize(f->ev_sv[d.side]));
  return fold_stage(f, d, true);
}

// Everything after the columns are on the device (on s_compute's dependency chain).
static bw_status run_batch(bw_fold* f, const u64* d_keys, const void* d_vals, const i64* d_ts, u64 rows, u64 epoch, Stage* stage) {
  bw_ctx* ctx = f->ctx;
  if (f->have_epoch && epoch < f->last_epoch) FAIL(f, BW_ERR_STATE, "epochs must not decrease (got %llu after %llu)", (unsigned long long)epoch, (unsigned long long)f->last_epoch);
  const u32 batch_no = f->batch_no++;
  if (!f->have_pending) { f->min_epoch = epoch; f->have_pending = true; }
  f->last_epoch = epoch;
  f->have_epoch = true;
  f->st.rows_ingested += rows;
  if (ctx->world == 1) f->st.rows_received += rows;
  Deferred d;
  d.side = (int)(batch_no & 1u);
  d.d_keys = d_keys;
  d.d_vals = d_vals;
  d.d_ts = d_ts;
  d.rows = rows;
  d.ord = epoch;
  d.batch_no = batch_no;
  d.stage = stage;
  const bool streamed = ctx->world > 1 ? f->stream_ok : stream_usable(f, d_keys, d_vals, d_ts, rows);
  bw_status st = BW_OK;
  if (streamed) {
    // queue this activation's scatter + verdict BEFORE looking at the previous verdict: the device
    // always has the next stage waiting while the host decides
    if ((st = stream_front(f, d_keys, d_vals, d_ts, rows, batch_no, d.side)) != BW_OK) return st;
    d.lanes = f->last_scatter_grid;  // (resolving the previous activation may scatter it a second time)
  }
  if ((st = stream_resolve(f)) != BW_OK) return st;  // activations fold in order
  if (streamed) {
    d.valid = true;
    f->dq = d;
  } else if ((st = fold_stage(f, d, false)) != BW_OK) {
    return st;
  }
  return flush_rows(f);
}

bw_status bw_ingest_commit(bw_fold* f, const bw_batch* batch, uint64_t rows, uint64_t epoch) {
  if (!f || !batch) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (f->eof_done) FAIL(f, BW_ERR_STATE, "commit after eof");
  f->host_ingest = true;
  if (batch->slot >= f->slots.size() || !f->slots[batch->slot].acquired) FAIL(f, BW_ERR_STATE, "commit of a slot that is not acquired");
  if (rows > f->spec.max_batch_rows) FAIL(f, BW_ERR_SPEC, "commit: rows > max_batch_rows");
  CU(ctx, cudaSetDevice(ctx->device));
  Slot& sl = f->slots[batch->slot];
  // device staging: 3 buffers, reused once the kernels that read them are done
  if (f->stages.empty()) f->stages.resize(3);
  Stage& sg = f->stages[f->stage_next];
  f->stage_next = (f->stage_next + 1) % (u32)f->stages.size();
  if (!sg.consumed) {  // (made last: a stage is complete once it has its event)
    const size_t cap = f->spec.max_batch_rows;
    CU(ctx, f->own.dev(&sg.d_keys, cap));
    if (f->has_vals) CU(ctx, f->own.dev(&sg.d_vals, cap * (size_t)f->val_bytes));
    if (f->has_ts) CU(ctx, f->own.dev(&sg.d_ts, cap));
    CU(ctx, f->own.event(&sg.consumed));
  }
  if (sg.used) CU(ctx, cudaStreamWaitEvent(f->s_copy, sg.consumed, 0));
  if (rows) {
    CU(ctx, cudaMemcpyAsync(sg.d_keys, sl.h_keys, rows * 8, cudaMemcpyHostToDevice, f->s_copy));
    if (f->has_vals) CU(ctx, cudaMemcpyAsync(sg.d_vals, sl.h_vals, rows * (size_t)f->val_bytes, cudaMemcpyHostToDevice, f->s_copy));
    if (f->has_ts) CU(ctx, cudaMemcpyAsync(sg.d_ts, sl.h_ts, rows * 8, cudaMemcpyHostToDevice, f->s_copy));
  }
  CU(ctx, cudaEventRecord(f->ev_h2d, f->s_copy));
  CU(ctx, cudaStreamWaitEvent(f->s_compute, f->ev_h2d, 0));
  f->cols_ready = f->ev_h2d;
  bw_status st = run_batch(f, sg.d_keys, sg.d_vals, sg.d_ts, rows, epoch, &sg);
  if (st != BW_OK) {  // (the slot goes back to the ring on the error paths too: repeated failures must not use it up)
    cudaEventSynchronize(f->ev_h2d);
    sl.acquired = false;
    return st;
  }
  // the pinned slot may be refilled once its H2D is done
  CU(ctx, cudaEventSynchronize(f->ev_h2d));
  sl.acquired = false;
  return BW_OK;
}

bw_status bw_ingest_device(bw_fold* f, const uint64_t* d_keys, const void* d_vals, const int64_t* d_ts_us, uint64_t rows,
                           uint64_t epoch) {
  if (!f) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (f->eof_done) FAIL(f, BW_ERR_STATE, "ingest after eof");
  if (rows > f->spec.max_batch_rows) FAIL(f, BW_ERR_SPEC, "ingest: rows > max_batch_rows");
  if (rows && (!d_keys || (!d_vals && (f->spec.reduction != BW_RED_COUNT || f->spec.ts_source == BW_TS_FROM_VALUE)) || (f->has_ts && !d_ts_us)))
    FAIL(f, BW_ERR_SPEC, "ingest: missing column");
  CU(ctx, cudaSetDevice(ctx->device));
  // The caller's columns are complete (bwgpu.h): the lateness pass and the exchange take no ordering from the fold's
  // stream, so they run beside the previous activation's fold instead of behind it.  Columns written by this
  // library's own generator are ordered through its event.
  f->cols_ready = f->ev_gen;
  return run_batch(f, d_keys, d_vals, d_ts_us, rows, epoch, nullptr);
}

// ---------------------------------------------------------------------------
// exact path for an activation with possible late items
// ---------------------------------------------------------------------------
struct MaxI64 {
  __host__ __device__ __forceinline__ i64 operator()(const i64& a, const i64& b) const { return a > b ? a : b; }
};

static bw_status slow_path(bw_fold* f, const BatchView& bv, u64 total, u64 epoch_ord, u32 batch_no) {
  bw_ctx* ctx = f->ctx;
  cudaStream_t s = f->s_compute;
  if (total == 0) return BW_OK;
  if (total > f->slow_cap) {
    CU(ctx, cudaStreamSynchronize(s));
    const u64 cap = std::max<u64>(total, 1024);
    Owner& own = f->own;
    f->slow_cap = 0;
    CU(ctx, own.regrow(Owner::DEV, &f->d_kflat, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_ksorted, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_tsflat, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_tssorted, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_prefmax, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_idx, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_idxsorted, cap));
    CU(ctx, own.regrow(Owner::DEV, &f->d_late, cap));
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, f->d_kflat, f->d_ksorted, f->d_idx, f->d_idxsorted, (int)cap, 0, 64, s);
    cub::DeviceScan::ExclusiveScanByKey(nullptr, b2, f->d_ksorted, f->d_tssorted, f->d_prefmax, MaxI64(), (i64)INT64_MIN,
                                        (int)cap, ::cuda::std::equal_to<>(), s);
    CU(ctx, f->srt.grow_cub(own, std::max(b1, b2) + 256));  // (the emission sort's CUB storage)
    f->slow_cap = cap;
  }
  const int grid = ctx->sm_count * 8;
  k_slow_flatten<<<grid, 256, 0, s>>>(bv, f->p, f->d_kflat, f->d_tsflat, f->d_idx);
  size_t tb = f->srt.cub_bytes;
  CU(ctx, cub::DeviceRadixSort::SortPairs(f->srt.cub, tb, f->d_kflat, f->d_ksorted, f->d_idx, f->d_idxsorted, (int)total, 0, 64, s));
  k_gather_i64<<<grid, 256, 0, s>>>(f->d_tsflat, f->d_idxsorted, f->d_tssorted, total);
  tb = f->srt.cub_bytes;
  CU(ctx, cub::DeviceScan::ExclusiveScanByKey(f->srt.cub, tb, f->d_ksorted, f->d_tssorted, f->d_prefmax, MaxI64(),
                                              (i64)INT64_MIN, (int)total, ::cuda::std::equal_to<>(), s));
  k_slow_classify<<<grid, 256, 0, s>>>(f->t, f->p, f->d_ksorted, f->d_idxsorted, f->d_tssorted, f->d_prefmax, f->d_late, total);
  k_slow_fold<<<f->fold_grid, BW_FOLD_THREADS, 0, s>>>(bv, f->t, f->p, f->e, f->d_late, batch_no, epoch_ord);
  CU(ctx, cudaGetLastError());
  f->st.kernel_launches += 4;  // ours; CUB's launches are not counted
  return BW_OK;
}

// ---------------------------------------------------------------------------
// advance / eof
// ---------------------------------------------------------------------------
// Build the reference-order permutation of n rows into x.perm (LSD passes of stable radix sorts).  A null `wid` skips
// the window-id pass.  The kernels this library launches are added to *launches, if given (CUB's are not counted).
static bw_status order_perm(bw_ctx* ctx, SortScratch& x, cudaStream_t s, u64 n, const u64* key, const u64* seq,
                            const u64* epoch, const i64* wid, u64 n_ordinals, u64 min_epoch, uint64_t* launches) {
  const int grid = ctx->sm_count * 4;
  k_iota<<<grid, 256, 0, s>>>(x.perm, n);
  struct Pass {
    int kind, bits;
  };
  int ebits = 1;
  while ((1ULL << ebits) < n_ordinals + 1) ++ebits;
  std::vector<Pass> passes;
  if (wid) passes.push_back({BW_SK_WID, 64});
  passes.push_back({BW_SK_SEQ, 64});
  passes.push_back({BW_SK_DIGITS, 16});
  passes.push_back({BW_SK_ALIGNED, 64});
  if (n_ordinals > 1) passes.push_back({BW_SK_EPOCH, ebits});
  if (launches) *launches += 1 + passes.size();
  for (const Pass& ps : passes) {
    k_sortkey<<<grid, 256, 0, s>>>(ps.kind, key, seq, epoch, wid, x.perm, x.sk, n, min_epoch);
    size_t tb = x.cub_bytes;
    CU(ctx, cub::DeviceRadixSort::SortPairs(x.cub, tb, x.sk, x.sk2, x.perm, x.perm2, (int)n, 0, ps.bits, s));
    std::swap(x.perm, x.perm2);
  }
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

static const char* status_name(u32 s) {
  switch (s) {
    case BW_ERR_CAPACITY: return "capacity exhausted (key table, pane pool, exchange region or emit buffer): raise capacity_hint / max_emit_rows / max_late_rows";
    case BW_ERR_RANGE: return "window id out of range (timestamp too far from align_to for this window length)";
    case BW_ERR_STATE: return "ordered fold with event time ahead of the system clock: at this notify phase the reference would "
                              "also wake keys at the timestamp of their oldest queued item, which the device does not keep";
    default: return "device-side failure";
  }
}

// Order rows [lo, hi) of the closed or late columns and copy them to the same positions of the host arrays.
static bw_status ship_rows(bw_fold* f, bool late, u64 lo, u64 hi, bool side) {
  bw_ctx* ctx = f->ctx;
  if (hi <= lo) return BW_OK;
  cudaStream_t s = side ? f->s_out : f->s_compute;
  const u64 n = hi - lo;
  const bool ordered = f->spec.emit_order == BW_ORDER_REFERENCE;
  const int grid = ctx->sm_count * 4;
  const u64 n_ord = f->have_pending ? (f->last_epoch - f->min_epoch + 1) : 1;
  // the window-id pass orders a key's rows where the sequence column ties: sliding windows emitted from one
  // pane, and folds whose sequence is just the closing activation (FoldParams::seq_by_id)
  const bool sliding = f->p.panes_per_window > 1 || f->p.panes_per_offset > 1 || f->p.seq_by_id;
  const EmitBufs& e = f->e;
  // (the side stream sorts in its own scratch: the main one is shared with the sort path of not-clean activations)
  SortScratch& x = side ? f->fl : f->srt;
  if (ordered) {
    if (side) CU(ctx, x.reserve(f->own, n, std::max<u64>(2 * n, 1 << 16), s));
    bw_status st;
    if (!late) st = order_perm(ctx, x, s, n, e.c_key + lo, e.c_seq + lo, e.c_epoch + lo, sliding ? e.c_wid + lo : nullptr, n_ord,
                               f->min_epoch, &f->st.kernel_launches);
    else  // rows of one late item were reserved contiguously in ascending window id; stable sorts keep that
      st = order_perm(ctx, x, s, n, e.l_key + lo, e.l_seq + lo, e.l_epoch + lo, nullptr, n_ord, f->min_epoch, &f->st.kernel_launches);
    if (st != BW_OK) return st;
  }
  // in the order of the host columns (bw_fold::ho_c, ho_l)
  const u64* cols[2][5] = {{e.c_key, (const u64*)e.c_wid, e.c_acc, e.c_count, e.c_epoch},
                           {e.l_key, (const u64*)e.l_wid, e.l_val, (const u64*)e.l_ts, e.l_epoch}};
  const u64* const* src = cols[late];
  u64* const* dst = late ? f->ho_l.col : f->ho_c.col;
  for (int c = 0; c < 5; ++c) {
    if (ordered) {
      k_gather_u64<<<grid, 256, 0, s>>>(src[c] + lo, x.perm, x.gather, n);
      f->st.kernel_launches++;
      CU(ctx, cudaMemcpyAsync(dst[c] + lo, x.gather, n * 8, cudaMemcpyDeviceToHost, s));
    } else {
      CU(ctx, cudaMemcpyAsync(dst[c] + lo, src[c] + lo, n * 8, cudaMemcpyDeviceToHost, s));
    }
  }
  return BW_OK;
}

// After an activation's fold stage has been queued: remember how many rows exist once it is done.
static bw_status mark_rows(bw_fold* f, u64 epoch) {
  bw_ctx* ctx = f->ctx;
  if (!f->flush_on || ctx->world > 1 || !f->host_ingest) return BW_OK;
  if (!f->s_out) {  // (the stream is made last: the side flush is ready once it exists)
    CU(ctx, f->own.host(&f->h_marks, 4 * 2));
    for (auto& m : f->marks) CU(ctx, f->own.event(&m.ev));
    CU(ctx, f->own.stream(&f->s_out));
  }
  if (f->mark_head) f->marks[(f->mark_head - 1) & 3].next_epoch = epoch + 1;  // (+1: 0 means "none yet")
  bw_fold::RowMark& m = f->marks[f->mark_head & 3];
  m.epoch = epoch;
  m.next_epoch = 0;
  m.live = true;
  CU(ctx, cudaMemcpyAsync(f->h_marks + 2 * (f->mark_head & 3), &f->d_ctr->n_closed, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                          f->s_compute));
  CU(ctx, cudaEventRecord(m.ev, f->s_compute));
  ++f->mark_head;
  return BW_OK;
}

// Rows of epochs that are closed -- a later activation with a larger epoch has been folded -- and whose counts have
// reached the host: order them and copy them out now, on the side stream, beside whatever the fold stream is doing.
// Segments end on epoch boundaries and are shipped in epoch order, so the host arrays end up exactly as one sort of
// everything would leave them (the order is epoch-major).
static bw_status flush_rows(bw_fold* f) {
  bw_ctx* ctx = f->ctx;
  if (!f->flush_on || !f->s_out) return BW_OK;
  for (u32 k = 0; k < 4 && k < f->mark_head; ++k) {  // newest first
    const u32 at = (f->mark_head - 1 - k) & 3;
    bw_fold::RowMark& m = f->marks[at];
    if (!m.live) break;
    if (!m.next_epoch || m.next_epoch - 1 <= m.epoch) continue;  // its epoch may still get rows
    if (cudaEventQuery(m.ev) != cudaSuccess) continue;
    const u64 nc = std::min<u64>(f->h_marks[2 * at], f->e.max_closed), nl = std::min<u64>(f->h_marks[2 * at + 1], f->e.max_late);
    bw_status st = ship_rows(f, false, f->done_c, nc, true);
    if (st != BW_OK) return st;
    st = ship_rows(f, true, f->done_l, nl, true);
    if (st != BW_OK) return st;
    if (nc > f->done_c) f->done_c = nc;
    if (nl > f->done_l) f->done_l = nl;
    for (u32 j = k; j < 4 && j < f->mark_head; ++j) f->marks[(f->mark_head - 1 - j) & 3].live = false;  // this one and the older ones: done
    CU(ctx, cudaGetLastError());
    break;
  }
  return BW_OK;
}

static bw_status collect(bw_fold* f, bw_emit* out) {
  bw_ctx* ctx = f->ctx;
  cudaStream_t s = f->s_compute;
  CU(ctx, cudaMemcpyAsync(f->h_ctr, f->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  if (f->s_out) CU(ctx, cudaStreamSynchronize(f->s_out));

  if (f->h_ctr->err) FAIL(f, (bw_status)f->h_ctr->err, "kernel raised status %u: %s", f->h_ctr->err, status_name(f->h_ctr->err));
  const u64 nc = std::min<u64>(f->h_ctr->n_closed, f->e.max_closed);
  const u64 nl = std::min<u64>(f->h_ctr->n_late, f->e.max_late);
  f->st.live_keys = f->h_ctr->live_keys;
  f->st.pane_nodes_used = f->h_ctr->pool_next - 1;
  CU(ctx, f->ho_c.reserve(f->own, nc, std::max<u64>(nc, 4096)));
  CU(ctx, f->ho_l.reserve(f->own, nl, std::max<u64>(nl, 4096)));
  bw_status st;
  // what the side stream has not already ordered and copied (everything, when nothing was flushed early)
  if ((st = ship_rows(f, false, std::min(f->done_c, nc), nc, false))) return st;
  if ((st = ship_rows(f, true, std::min(f->done_l, nl), nl, false))) return st;
  f->done_c = f->done_l = 0;
  for (auto& m : f->marks) m.live = false;
  // reset the row counters for the next round
  CU(ctx, cudaMemsetAsync(&f->d_ctr->n_closed, 0, sizeof(unsigned long long) * 2, s));
  CU(ctx, cudaStreamSynchronize(s));
  f->have_pending = false;
  out->n_closed = nc;
  out->closed_key = f->ho_c.col[0];
  out->closed_window_id = (i64*)f->ho_c.col[1];
  out->closed_acc = f->ho_c.col[2];
  out->closed_count = f->ho_c.col[3];
  out->closed_epoch = f->ho_c.col[4];
  out->n_late = nl;
  out->late_key = f->ho_l.col[0];
  out->late_window_id = (i64*)f->ho_l.col[1];
  out->late_val = f->ho_l.col[2];
  out->late_ts_us = (i64*)f->ho_l.col[3];
  out->late_epoch = f->ho_l.col[4];
  return BW_OK;
}

bw_status bw_fold_set_system_now(bw_fold* f, int64_t system_now_us) {
  if (!f) return BW_ERR_SPEC;
  if (f->ctx->world > 1) FAIL(f, BW_ERR_SPEC, "bw_fold_set_system_now: one rank only (every rank would need the same clock)");
  CU(f->ctx, cudaSetDevice(f->ctx->device));
  if (!f->p.track_wm || f->p.ts_from_value == 2) return BW_OK;  // no watermark to move
  if (system_now_us <= f->p.now_us) return BW_OK;              // "don't let now go backwards" (windowing.py:250-261)
  bw_status st = stream_resolve(f);  // the activation in flight was scattered in the old frame: fold it there
  if (st != BW_OK) return st;
  f->p.now_us = system_now_us;
  f->p.align_us = f->spec.align_to_us - system_now_us;
  return BW_OK;
}

bw_status bw_advance(bw_fold* f, uint64_t closed_epoch, int64_t system_now_us, bw_emit* out) {
  (void)closed_epoch;
  if (!f || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = stream_resolve(f);
  if (st != BW_OK) return st;
  if (system_now_us > 0 && ctx->world == 1 && f->p.track_wm && f->p.ts_from_value != 2 && !f->eof_done) {
    // the notify phase at this system time: due keys close what their watermark now allows
    st = bw_fold_set_system_now(f, system_now_us);
    if (st != BW_OK) return st;
    if (!f->have_pending) { f->min_epoch = f->last_epoch; f->have_pending = true; }
    k_close_wake<<<f->close_grid, 256, 0, f->s_compute>>>(f->t, f->p, f->e, f->last_epoch, f->batch_no);
    CU(ctx, cudaGetLastError());
    f->st.kernel_launches++;
  }
  return collect(f, out);
}

bw_status bw_eof(bw_fold* f, bw_emit* out) {
  if (!f || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (f->eof_done) FAIL(f, BW_ERR_STATE, "eof called twice");
  {
    bw_status st = stream_resolve(f);
    if (st != BW_OK) return st;
  }
  const u64 ord = f->last_epoch;
  if (!f->have_pending) { f->min_epoch = f->last_epoch; f->have_pending = true; }
  k_close_all<<<f->close_grid, 256, 0, f->s_compute>>>(f->t, f->p, f->e, ord, f->batch_no);
  CU(ctx, cudaGetLastError());
  f->st.kernel_launches++;
  f->eof_done = true;
  return collect(f, out);
}

// ---------------------------------------------------------------------------
// snapshot / restore
// ---------------------------------------------------------------------------
static SnapCols snap_cols(void* base, u64 n) {
  SnapCols c;
  u64* b = (u64*)base;
  c.key = b;
  c.pane = (i64*)(b + n);
  c.acc = b + 2 * n;
  c.cnt = b + 3 * n;
  c.seq = b + 4 * n;
  c.max_ts = (i64*)(b + 5 * n);
  c.closed_upto = (i64*)(b + 6 * n);
  c.cap = n;
  return c;
}

bw_status bw_snapshot_take(bw_fold* f, bw_snapshot* out) {
  if (!f || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (f->eof_done) FAIL(f, BW_ERR_STATE, "snapshot after eof");
  {
    bw_status st = stream_resolve(f);
    if (st != BW_OK) return st;
  }
  cudaStream_t s = f->s_compute;
  if (f->s_x) CU(ctx, cudaStreamSynchronize(f->s_x));
  if (!f->d_snap_ctr) CU(ctx, f->own.dev(&f->d_snap_ctr, 2));
  CU(ctx, cudaMemsetAsync(f->d_snap_ctr, 0, 2 * sizeof(unsigned long long), s));
  k_snap_count<<<f->close_grid, 256, 0, s>>>(f->t, f->d_snap_ctr);
  unsigned long long n = 0;
  CU(ctx, cudaMemcpyAsync(&n, f->d_snap_ctr, sizeof n, cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaMemcpyAsync(f->h_ctr, f->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  if (f->h_ctr->err) FAIL(f, (bw_status)f->h_ctr->err, "a kernel reported status %u before the snapshot", f->h_ctr->err);
  const u64 rows = n ? n : 1;
  CU(ctx, f->own.regrow(Owner::DEV, &f->snap_dev, rows * 7 * 8));
  CU(ctx, f->own.regrow(Owner::HOST, &f->snap_host, rows * 7 * 8));
  SnapCols dc = snap_cols(f->snap_dev, rows), hc = snap_cols(f->snap_host, rows);
  if (n) {
    FoldParams p0 = f->p;  // the frame of system time 0, the one a restoring fold loads in
    p0.align_us = f->spec.align_to_us;
    k_snap_fill<<<f->close_grid, 256, 0, s>>>(f->t, p0, dc, f->d_snap_ctr + 1);
    CU(ctx, cudaGetLastError());
    CU(ctx, cudaMemcpyAsync(f->snap_host, f->snap_dev, rows * 7 * 8, cudaMemcpyDeviceToHost, s));
    CU(ctx, cudaStreamSynchronize(s));
  }
  f->st.kernel_launches += n ? 2 : 1;
  memset(out, 0, sizeof *out);
  out->n = n;
  out->key = hc.key;
  out->pane_id = hc.pane;
  out->acc = hc.acc;
  out->count = hc.cnt;
  out->open_seq = hc.seq;
  out->max_ts_us = hc.max_ts;
  out->closed_upto = hc.closed_upto;
  out->batch_no = f->batch_no;
  out->gmax_ts_us = (i64)f->h_ctr->gmax_ts;
  out->last_epoch = f->last_epoch;
  return BW_OK;
}

bw_status bw_snapshot_load(bw_fold* f, const bw_snapshot* in) {
  if (!f || !in) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (f->batch_no != 0 || f->eof_done) FAIL(f, BW_ERR_STATE, "bw_snapshot_load needs a freshly created fold");
  if (in->n && (!in->key || !in->pane_id || !in->acc || !in->count || !in->open_seq || !in->max_ts_us || !in->closed_upto))
    FAIL(f, BW_ERR_SPEC, "bw_snapshot_load: missing column");
  if (in->batch_no >= (1ULL << 32)) FAIL(f, BW_ERR_SPEC, "bw_snapshot_load: bad batch_no");
  cudaStream_t s = f->s_compute;
  const u64 n = in->n;
  if (n) {
    CU(ctx, f->own.regrow(Owner::DEV, &f->snap_dev, n * 7 * 8));
    SnapCols dc = snap_cols(f->snap_dev, n);
    const void* src[7] = {in->key, in->pane_id, in->acc, in->count, in->open_seq, in->max_ts_us, in->closed_upto};
    void* dst[7] = {dc.key, dc.pane, dc.acc, dc.cnt, dc.seq, dc.max_ts, dc.closed_upto};
    for (int c = 0; c < 7; ++c) CU(ctx, cudaMemcpyAsync(dst[c], src[c], n * 8, cudaMemcpyHostToDevice, s));
    k_snap_load<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(f->t, f->p, dc, n, (u32)in->batch_no, ctx->world, ctx->rank);
    CU(ctx, cudaGetLastError());
    // re-rank every restored key (newest pane into the hot slot); nothing is closable in a state dumped after an advance
    k_close_dirty<<<f->close_grid, 256, 0, s>>>(f->t, f->p, f->e, in->last_epoch, (u32)in->batch_no);
    k_reset_dirty<<<1, 1, 0, s>>>(f->t);
    f->st.kernel_launches += 3;
    CU(ctx, cudaStreamSynchronize(s));
  }
  k_snap_set_gmax<<<1, 1, 0, s>>>(f->d_ctr, (i64)in->gmax_ts_us);
  CU(ctx, cudaMemcpyAsync(f->h_ctr, f->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  if (f->h_ctr->err) FAIL(f, (bw_status)f->h_ctr->err, "restore failed on the device with status %u (capacity_hint too small?)", f->h_ctr->err);
  f->batch_no = (u32)in->batch_no;
  f->h_gmax = std::max<i64>(f->h_gmax, (i64)in->gmax_ts_us);
  f->last_epoch = in->last_epoch;
  f->have_epoch = in->last_epoch != 0;
  return BW_OK;
}

void bw_window_bounds(const bw_fold_spec* spec, int64_t window_id, int64_t* open_us, int64_t* close_us) {
  const int64_t o = spec->align_to_us + spec->offset_us * window_id;
  if (open_us) *open_us = o;
  if (close_us) *close_us = o + spec->length_us;
}

static void drain_timers(bw_fold* f) {
  for (size_t i = 0; i < f->timers_used; ++i) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, f->timers[i].a, f->timers[i].b) == cudaSuccess) {
      if (f->timers[i].kind == 1) {
        f->st.sum_scatter_ms += ms;
        f->st.scatter_launches++;
      } else if (f->timers[i].kind == 2) {
        f->st.sum_verdict_ms += ms;
      } else {
        f->st.last_fold_ms = ms;
        f->st.sum_fold_ms += ms;
        f->st.fold_rows += f->timers[i].rows;
        f->st.timed_folds++;
      }
    }
  }
  f->timers_used = 0;
}

bw_status bw_fold_stats(bw_fold* f, bw_stats* out) {
  if (!f || !out) return BW_ERR_SPEC;
  CU(f->ctx, cudaSetDevice(f->ctx->device));
  {
    bw_status st = stream_resolve(f);
    if (st != BW_OK) return st;
  }
  CU(f->ctx, cudaStreamSynchronize(f->s_compute));
  drain_timers(f);
  *out = f->st;
  return BW_OK;
}
bw_status bw_fold_reset_timers(bw_fold* f) {
  if (!f) return BW_ERR_SPEC;
  {
    bw_status st = stream_resolve(f);
    if (st != BW_OK) return st;
  }
  CU(f->ctx, cudaStreamSynchronize(f->s_compute));
  drain_timers(f);
  f->st.sum_scatter_ms = 0;
  f->st.sum_verdict_ms = 0;
  f->st.scatter_launches = 0;
  f->st.sum_fold_ms = 0;
  f->st.last_fold_ms = 0;
  f->st.fold_rows = 0;
  f->st.timed_folds = 0;
  f->st.fold_launches = 0;
  f->st.combined_folds = 0;
  f->st.split_batches = 0;
  return BW_OK;
}
// Fold the deferred activation, then wait for the copy, lateness and exchange streams, and for the fold's own stream
// too when `compute`.
static bw_status resolve_and_sync(bw_fold* f, bool compute) {
  bw_status st = stream_resolve(f);
  if (st != BW_OK) return st;
  for (cudaStream_t s : {f->s_copy, f->s_pre, f->s_x}) CU(f->ctx, cudaStreamSynchronize(s));
  if (compute) CU(f->ctx, cudaStreamSynchronize(f->s_compute));
  return BW_OK;
}
bw_status bw_fold_sync(bw_fold* f) {
  if (!f) return BW_ERR_SPEC;
  CU(f->ctx, cudaSetDevice(f->ctx->device));
  return resolve_and_sync(f, true);
}

bw_status bw_fold_set_segfold_parts(bw_fold* f, uint32_t parts) {
  if (!f) return BW_ERR_SPEC;
  if (parts & ~BW_SF_ALL) FAIL(f, BW_ERR_SPEC, "bw_fold_set_segfold_parts: unknown bits 0x%x", parts & ~BW_SF_ALL);
  f->segfold_parts = parts;
  return BW_OK;
}

// out[0]: slots (the alias slot included) whose dense key differs from hot[].key, out[1]: slots holding a key
__global__ void k_check_key_column(Table t, unsigned long long* out) {
  unsigned long long bad = 0, used = 0;
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.cap; s += (u64)gridDim.x * blockDim.x) {
    const u64 k = t.hot[s].key;
    bad += t.keys[s] != k;
    used += k != BW_EMPTY_KEY;
  }
  if (bad) atomicAdd(out, bad);
  if (used) atomicAdd(out + 1, used);
}

bw_status bw_fold_check_key_column(bw_fold* f, uint64_t* mismatches, uint64_t* keys) {
  if (!f || !mismatches || !keys) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = resolve_and_sync(f, true);
  if (st != BW_OK) return st;
  cudaStream_t s = f->s_compute;
  if (!f->d_snap_ctr) CU(ctx, f->own.dev(&f->d_snap_ctr, 2));  // (the snapshot's two counters: free between calls)
  CU(ctx, cudaMemsetAsync(f->d_snap_ctr, 0, 2 * sizeof(unsigned long long), s));
  k_check_key_column<<<ctx->sm_count * 4, 256, 0, s>>>(f->t, f->d_snap_ctr);
  CU(ctx, cudaGetLastError());
  unsigned long long h[2];
  CU(ctx, cudaMemcpyAsync(h, f->d_snap_ctr, sizeof h, cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  *mismatches = h[0];
  *keys = h[1];
  return BW_OK;
}
bw_status bw_fold_time_begin(bw_fold* f) {
  if (!f) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (!f->ev_t0) {
    CU(ctx, f->own.event(&f->ev_t0, cudaEventDefault));
    CU(ctx, f->own.event(&f->ev_t1, cudaEventDefault));
  }
  // everything submitted so far (copies, prepass) must be done before the clock starts
  bw_status st = resolve_and_sync(f, true);
  if (st != BW_OK) return st;
  CU(ctx, cudaEventRecord(f->ev_t0, f->s_compute));
  return BW_OK;
}
bw_status bw_fold_time_end(bw_fold* f, float* ms) {
  if (!f || !ms || !f->ev_t0) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  bw_status st = resolve_and_sync(f, false);  // (the fold's stream ends in the record below)
  if (st != BW_OK) return st;
  CU(ctx, cudaEventRecord(f->ev_t1, f->s_compute));
  CU(ctx, cudaEventSynchronize(f->ev_t1));
  CU(ctx, cudaEventElapsedTime(ms, f->ev_t0, f->ev_t1));
  return BW_OK;
}
void* bw_fold_stream(bw_fold* f) { return f ? (void*)f->s_compute : nullptr; }

bw_status bw_gen_c1(bw_fold* f, uint64_t* d_keys, uint64_t* d_vals, uint64_t start, uint64_t rows, uint64_t n_keys) {
  if (!f || !n_keys) return BW_ERR_SPEC;
  CU(f->ctx, cudaSetDevice(f->ctx->device));
  k_gen_c1<<<f->ctx->sm_count * 8, 256, 0, f->s_compute>>>(d_keys, d_vals, start, rows, n_keys);
  CU(f->ctx, cudaGetLastError());
  if (!f->ev_gen) CU(f->ctx, f->own.event(&f->ev_gen));
  CU(f->ctx, cudaEventRecord(f->ev_gen, f->s_compute));
  f->st.kernel_launches++;
  return BW_OK;
}


// ===========================================================================
// K5 / K6 host side
// ===========================================================================
struct MaxU32 {
  __host__ __device__ __forceinline__ u32 operator()(const u32& a, const u32& b) const { return a > b ? a : b; }
};

struct KeyedScratch {  // grouping of one activation by key (stable)
  u64 cap = 0;
  u64 *d_keys = nullptr, *d_ksorted = nullptr, *d_slot = nullptr;
  u32 *d_idx = nullptr, *d_isorted = nullptr, *d_head = nullptr;
  void* d_cub = nullptr;
  size_t cub_bytes = 0;
};

static bw_status keyed_alloc(bw_ctx* ctx, Owner& own, KeyedScratch& k, u64 cap, cudaStream_t s) {
  k.cap = cap;
  CU(ctx, own.dev(&k.d_keys, cap));
  CU(ctx, own.dev(&k.d_ksorted, cap));
  CU(ctx, own.dev(&k.d_slot, cap));
  CU(ctx, own.dev(&k.d_idx, cap));
  CU(ctx, own.dev(&k.d_isorted, cap));
  CU(ctx, own.dev(&k.d_head, cap));
  size_t b1 = 0, b2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b1, k.d_keys, k.d_ksorted, k.d_idx, k.d_isorted, (int)cap, 0, 64, s);
  cub::DeviceScan::InclusiveScan(nullptr, b2, k.d_head, k.d_head, MaxU32(), (int)cap, s);
  k.cub_bytes = std::max(b1, b2) + 256;
  CU(ctx, own.dev(&k.d_cub, k.cub_bytes));
  return BW_OK;
}
// stable group-by-key of n device keys: ksorted / isorted / head positions
static bw_status keyed_group(bw_ctx* ctx, KeyedScratch& k, const u64* d_keys, u64 n, cudaStream_t s) {
  const int grid = ctx->sm_count * 4;
  k_iota<<<grid, 256, 0, s>>>(k.d_idx, n);
  size_t tb = k.cub_bytes;
  CU(ctx, cub::DeviceRadixSort::SortPairs(k.d_cub, tb, d_keys, k.d_ksorted, k.d_idx, k.d_isorted, (int)n, 0, 64, s));
  k_keyed_heads<<<grid, 256, 0, s>>>(k.d_ksorted, k.d_head, n);
  tb = k.cub_bytes;
  CU(ctx, cub::DeviceScan::InclusiveScan(k.d_cub, tb, k.d_head, k.d_head, MaxU32(), (int)n, s));
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

// ---- keyed kernels on N ranks (K5, K6, K7, K8): every row to its key's owner ----
// One rank's receive region: a 256-byte head of four rows of BW_MAX_WORLD u64 -- per source rank r: the rows r sent
// here, the epoch, the system time and the refusal flag r published (k_xchg_head) -- then source r's keys, values and ts
// (8 bytes each, the partition's column widths), with source rows its rows' indices (4 bytes) and, with sides, its
// rows' sides (1 byte; K8) at [r * cap].  With a return section (a keyed map, K5), 256-byte aligned at the end: this rank's own `cap` rows of mu (f64), sigma (f64),
// the W owners' error words (u32, BW_MAX_WORLD of them) and flag (u8), which owners store into at the row's index.
// Setup is collective: the region is shared with every rank (coll_share_base).  A call is collective too: send()
// publishes the head, partitions the source's columns straight into the owners' regions (peer stores), enters a barrier
// and reads the head; the caller checks it, gathers what arrived (and, with a return section, maps it and stores the
// results back), then done() enters a second barrier, past which no source of the next call overwrites rows an owner
// still reads, and every source may read its return section.  A second barrier rather than double-buffered regions: a
// call already waits on the host for the received counts, so a second region set would leave nothing to overlap and
// would double the region.
#define BW_XRET_ROW_BYTES 17  // mu, sigma, flag
struct RankXchg {
  u64 cap = 0;       // rows per source: max_batch_rows
  bool src_rows = false, sides = false;
  size_t keys_off = 0, vals_off = 0, ts_off = 0, rows_off = 0, side_off = 0, ret_off = 0, total = 0;
  int ret_row = 0;   // bytes of a return row: 0 (none) or BW_XRET_ROW_BYTES
  void* base = nullptr;
  void* peer[BW_MAX_WORLD] = {nullptr};  // every rank's region as seen from here
  u32* d_tile_counts = nullptr;
  Counters* d_ctr = nullptr;  // k_part_scan's error word: never raised, a source sends at most `cap` rows
  u32* d_word = nullptr;      // coll_barrier's word
  u64* h_head = nullptr;      // pinned: the head as received

  // with_sides needs with_src_rows (k_part_scatter<true, true>)
  bw_status setup(bw_ctx* ctx, Owner& own, u64 max_batch_rows, bool with_src_rows, bool with_sides, int ret_row_bytes, cudaStream_t s) {
    if (ret_row_bytes != 0 && ret_row_bytes != BW_XRET_ROW_BYTES) CTX_FAIL(ctx, BW_ERR_SPEC, "RankXchg: bad return row width");
    if (with_sides && !with_src_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "RankXchg: sides travel only with source rows");
    cap = max_batch_rows;
    src_rows = with_src_rows;
    sides = with_sides;
    ret_row = ret_row_bytes;
    const size_t col = (size_t)cap * ctx->world;
    keys_off = 4 * BW_MAX_WORLD * sizeof(u64);
    vals_off = keys_off + col * 8;
    ts_off = vals_off + col * 8;
    rows_off = ts_off + col * 8;
    side_off = rows_off + (src_rows ? col * 4 : 0);
    total = side_off + (sides ? col : 0);
    if (ret_row) {
      ret_off = (total + 255) & ~(size_t)255;
      total = ret_off + (size_t)cap * ret_row + BW_MAX_WORLD * sizeof(u32);
    }
    CU(ctx, own.dev(&base, total));
    if (ret_row) CU(ctx, cudaMemsetAsync(ret_at(base).err, 0, BW_MAX_WORLD * sizeof(u32), s));
    CU(ctx, own.dev(&d_tile_counts, ((cap + BW_PART_TILE - 1) / BW_PART_TILE + 1) * BW_MAX_WORLD));
    CU(ctx, own.dev(&d_ctr, 1));
    CU(ctx, own.dev(&d_word, 1));
    CU(ctx, own.host(&h_head, 4 * BW_MAX_WORLD));
    CU(ctx, cudaMemsetAsync(d_ctr, 0, sizeof(Counters), s));
    CU(ctx, cudaMemsetAsync(d_word, 0, 4, s));
    CU(ctx, cudaFuncSetAttribute(sides ? k_part_scatter<true, true> : src_rows ? k_part_scatter<true> : k_part_scatter<false>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, BW_PART_TILE * (sides ? 29 : src_rows ? 28 : 24)));
    CU(ctx, cudaStreamSynchronize(s));
    return coll_share_base(ctx, base, peer, s);
  }
  // closes the IPC mappings; the caller's Owner frees the rest
  void close(bw_ctx* ctx) {
    for (int r = 0; r < ctx->world; ++r)
      if (r != ctx->rank && !ctx->loop && peer[r]) cudaIpcCloseMemHandle(peer[r]);
  }
  // head row `row` (0 rows, 1 epoch, 2 system time, 3 refusal flag), one entry per source rank
  const u64* head(int row) const { return h_head + row * BW_MAX_WORLD; }
  // `side`: the source's side column, set up with sides (it may be NULL when in.n is 0)
  bw_status send(bw_ctx* ctx, cudaStream_t s, const PartIn& in, u64 epoch, i64 now, bool refused, const unsigned char* side = nullptr) {
    const int W = ctx->world, R = ctx->rank;
    PartOut po;
    memset(&po, 0, sizeof po);
    po.region_cap = cap;
    PartSide ps;
    memset(&ps, 0, sizeof ps);
    ps.src = side;
    XchgHead pub;
    for (int d = 0; d < W; ++d) {
      char* b = (char*)peer[d];
      po.counts[d] = (u64*)b + R;
      pub.at[d] = (u64*)b + R;
      po.keys[d] = (u64*)(b + keys_off) + (size_t)R * cap;
      po.vals[d] = (u64*)(b + vals_off) + (size_t)R * cap;
      po.ts[d] = (i64*)(b + ts_off) + (size_t)R * cap;
      if (src_rows) po.rows[d] = (u32*)(b + rows_off) + (size_t)R * cap;
      if (sides) ps.dst[d] = (unsigned char*)(b + side_off) + (size_t)R * cap;
    }
    const u64 ntiles = (in.n + BW_PART_TILE - 1) / BW_PART_TILE;
    const int grid = (int)std::min<u64>(std::max<u64>(ntiles, 1), (u64)ctx->sm_count * 8);
    const size_t stage = (size_t)BW_PART_TILE * (8 + in.val_bytes + (in.ts ? 8 : 0) + (src_rows ? 4 : 0) + (sides ? 1 : 0));
    k_xchg_head<<<1, 32, 0, s>>>(pub, W, epoch, now, refused ? 1 : 0);
    k_part_hist<<<grid, BW_PART_THREADS, 0, s>>>(in, d_tile_counts);
    k_part_scan<<<W, 1024, 0, s>>>(in.n, W, d_tile_counts, po, d_ctr);
    if (sides) k_part_scatter<true, true><<<grid, BW_PART_THREADS, stage, s>>>(in, d_tile_counts, po, ps);
    else if (src_rows) k_part_scatter<true><<<grid, BW_PART_THREADS, stage, s>>>(in, d_tile_counts, po, ps);
    else k_part_scatter<false><<<grid, BW_PART_THREADS, stage, s>>>(in, d_tile_counts, po, ps);
    CU(ctx, cudaGetLastError());
    // every rank's stores are complete once it enters the barrier (stream order)
    bw_status st = coll_barrier(ctx, d_word, s);
    if (st != BW_OK) return st;
    CU(ctx, cudaMemcpyAsync(h_head, base, sizeof(u64) * 4 * BW_MAX_WORLD, cudaMemcpyDeviceToHost, s));
    CU(ctx, cudaStreamSynchronize(s));
    return BW_OK;
  }
  // the received segments, in source rank order; returns the rows in all of them
  u64 received(bw_ctx* ctx, BatchView& bv) const {
    memset(&bv, 0, sizeof bv);
    u64 n = 0;
    for (int r = 0; r < ctx->world; ++r) {
      const char* b = (const char*)base;
      bv.keys[r] = (const u64*)(b + keys_off) + (size_t)r * cap;
      bv.vals[r] = (const u64*)(b + vals_off) + (size_t)r * cap;
      bv.ts[r] = (const i64*)(b + ts_off) + (size_t)r * cap;
      bv.h_counts[r] = h_head[r];
      n += h_head[r];
    }
    bv.nseg = ctx->world;
    return n;
  }
  const u32* rows() const { return (const u32*)((const char*)base + rows_off); }
  const unsigned char* side() const { return (const unsigned char*)base + side_off; }
  bw_status done(bw_ctx* ctx, cudaStream_t s) { return coll_barrier(ctx, d_word, s); }
  // the return section of the region at `b` (setup with a return row width)
  XchgRet ret_at(void* b) const {
    char* p = (char*)b + ret_off;
    XchgRet c;
    c.mu = (double*)p;
    c.sigma = (double*)(p + cap * 8);
    c.err = (u32*)(p + cap * 16);
    c.flag = (unsigned char*)(c.err + BW_MAX_WORLD);
    return c;
  }
  XchgRet ret_mine() const { return ret_at(base); }
  XchgRetPeers ret_peers(bw_ctx* ctx) const {
    XchgRetPeers p;
    memset(&p, 0, sizeof p);
    for (int r = 0; r < ctx->world; ++r) p.at[r] = ret_at(peer[r]);
    return p;
  }
};

struct bw_smap {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_smap_spec spec{};
  SmapTable t{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;
  void* d_vals = nullptr;
  double *d_mu = nullptr, *d_sigma = nullptr;
  unsigned char* d_flag = nullptr;
  // sharded by key (shard_by_key on world > 1): the exchange (with source rows and a return section), each gathered
  // row's name (source rank << 32 | source row), the owners' error words as read back, and whether a call has failed
  bool shard = false;
  RankXchg x;
  u64* d_name = nullptr;
  u32* h_ret_err = nullptr;
  bool failed = false;
};

bw_status bw_smap_create(bw_ctx* ctx, const bw_smap_spec* user, bw_smap** out) {
  if (!ctx || !user || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_smap_create: NULL argument");
  // a spec built against the header before shard_by_key existed ends just before it, and leaves it 0
  if (user->struct_size != sizeof(bw_smap_spec) && user->struct_size != offsetof(bw_smap_spec, shard_by_key))
    CTX_FAIL(ctx, BW_ERR_SPEC, "bw_smap_spec.struct_size mismatch");
  bw_smap_spec copy{};
  memcpy(&copy, user, user->struct_size);
  const bw_smap_spec* spec = &copy;
  if (spec->window < 1 || spec->window > BW_SMAP_MAXW) CTX_FAIL(ctx, BW_ERR_SPEC, "window must be in 1..%d", BW_SMAP_MAXW);
  if (spec->val_dtype != BW_VAL_F32 && spec->val_dtype != BW_VAL_F64) CTX_FAIL(ctx, BW_ERR_SPEC, "val_dtype must be F32 or F64");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  const bool shard = spec->shard_by_key && ctx->world > 1;
  // an owner groups up to max_batch_rows from every rank with 32-bit sort indices, and names rows rank << 32 | row
  if (shard && spec->max_batch_rows > ((1ULL << 31) - 1) / (u64)ctx->world)
    CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows: max_batch_rows * world must be in [1, 2^31)");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_smap, void (*)(bw_smap*)> mp(new bw_smap(), bw_smap_destroy);  // torn down on every failure
  bw_smap* m = mp.get();
  Owner& own = m->own;
  m->ctx = ctx;
  m->spec = *spec;
  m->shard = shard;
  u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  m->t.cap = cap;
  m->t.window = spec->window;
  CU(ctx, own.stream(&m->s));
  CU(ctx, own.dev(&m->t.keys, cap + 1));
  CU(ctx, own.dev(&m->t.cnt, cap + 1));
  CU(ctx, own.dev(&m->t.ring, (cap + 1) * (u64)spec->window));
  CU(ctx, own.dev(&m->t.err, 1));
  CU(ctx, cudaMemsetAsync(m->t.err, 0, 4, m->s));
  CU(ctx, own.host(&m->h_err, 64 / sizeof(u32)));
  // rows one activation brings to this rank: its own, or up to max_batch_rows from every rank when sharded
  const u64 n = spec->max_batch_rows * (shard ? (u64)ctx->world : 1);
  bw_status st = keyed_alloc(ctx, own, m->k, n, m->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&m->d_vals, n * 8));
  CU(ctx, own.dev(&m->d_mu, n));
  CU(ctx, own.dev(&m->d_sigma, n));
  CU(ctx, own.dev(&m->d_flag, n));
  k_smap_init<<<ctx->sm_count * 4, 256, 0, m->s>>>(m->t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(m->s));
  if (shard) {
    CU(ctx, own.dev(&m->d_name, n));
    CU(ctx, own.host(&m->h_ret_err, BW_MAX_WORLD));
    st = m->x.setup(ctx, own, spec->max_batch_rows, true, false, BW_XRET_ROW_BYTES, m->s);
    if (st != BW_OK) return st;
  }
  *out = mp.release();
  return BW_OK;
}

void bw_smap_destroy(bw_smap* m) {
  if (!m) return;
  cudaSetDevice(m->ctx->device);
  if (m->s) cudaStreamSynchronize(m->s);
  m->x.close(m->ctx);
  delete m;  // m->own releases every buffer and the stream
}

// K5 over n device rows: group by key, then the ring kernels; outputs aligned with the rows
static bw_status smap_map(bw_smap* m, const u64* d_keys, const void* d_vals, u64 n, double* d_mu, double* d_sigma, uint8_t* d_flag) {
  bw_ctx* ctx = m->ctx;
  bw_status st = keyed_group(ctx, m->k, d_keys, n, m->s);
  if (st != BW_OK) return st;
  const int grid = ctx->sm_count * 8;
  const int is_f32 = m->spec.val_dtype == BW_VAL_F32;
  k_smap_slots<<<grid, 256, 0, m->s>>>(m->t, m->k.d_ksorted, m->k.d_head, m->k.d_slot, n);
  k_smap_eval<<<grid, 256, 0, m->s>>>(m->t, m->k.d_isorted, m->k.d_head, m->k.d_slot, d_vals, is_f32, m->spec.threshold, d_mu, d_sigma,
                                       d_flag, n);
  k_smap_update<<<grid, 256, 0, m->s>>>(m->t, m->k.d_ksorted, m->k.d_isorted, m->k.d_head, m->k.d_slot, d_vals, is_f32, n);
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

// bw_smap_apply / _apply_device when sharded by key (include/bwgpu.h): every row to its key's owner, K5 there over
// what arrived, and each row's mu, sigma and flag back to its source rank at its row.  `host`: the columns are host
// memory.  Blocks until the call is complete.
static bw_status smap_apply_ranks(bw_smap* m, const u64* keys, const void* vals, u64 rows, double* mu, double* sigma, uint8_t* flag,
                                  bool host) {
  bw_ctx* ctx = m->ctx;
  const int W = ctx->world;
  const int is_f32 = m->spec.val_dtype == BW_VAL_F32;
  cudaStream_t s = m->s;
  CU(ctx, cudaSetDevice(ctx->device));
  // A call that cannot go ahead still takes part in the exchange and both barriers, so that no peer waits for it in a
  // barrier: it sends no rows and raises its refusal flag, and every rank then fails the call.
  bw_status refuse = BW_OK;
  const char* why = "";
  if (m->failed) {
    refuse = BW_ERR_STATE;
    why = "smap: an earlier call failed; the map is unusable";
  } else if (rows > m->spec.max_batch_rows) {
    refuse = BW_ERR_SPEC;
    why = "smap: rows > max_batch_rows";
  } else if (rows && (!keys || !vals || !mu || !sigma || !flag)) {
    refuse = BW_ERR_SPEC;
    why = "smap: NULL column";
  }
  if (refuse != BW_OK) rows = 0;
  PartIn in;
  in.keys = keys;
  in.vals = vals;
  in.ts = nullptr;
  in.n = rows;
  in.val_bytes = is_f32 ? 4 : 8;
  in.world = W;
  if (host && rows) {  // staged in K5's own columns: the gather overwrites them only after the scatter has read them
    CU(ctx, cudaMemcpyAsync(m->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(m->d_vals, vals, rows * in.val_bytes, cudaMemcpyHostToDevice, s));
    in.keys = m->k.d_keys;
    in.vals = m->d_vals;
  }
  // K5 has no epoch and no clock: the head's epoch and time rows carry 0
  bw_status st = m->x.send(ctx, s, in, 0, 0, refuse != BW_OK);
  if (st != BW_OK) return st;
  // every rank reads the same head: all of them fail here, or none does
  const u64* got_refused = m->x.head(3);
  int refused = -1;
  for (int r = W - 1; r >= 0; --r)
    if (got_refused[r]) refused = r;
  if (refused < 0) {
    BatchView bv;
    const u64 n = m->x.received(ctx, bv);
    if (n) {
      k_xsmap_gather<<<ctx->sm_count * 4, 256, 0, s>>>(bv, m->x.rows(), m->spec.max_batch_rows, n, is_f32, m->k.d_keys, m->d_vals, m->d_name);
      CU(ctx, cudaGetLastError());
      st = smap_map(m, m->k.d_keys, m->d_vals, n, m->d_mu, m->d_sigma, m->d_flag);
      if (st != BW_OK) return st;
    }
    k_xsmap_return<<<ctx->sm_count * 4, 256, 0, s>>>(m->x.ret_peers(ctx), m->d_name, m->d_mu, m->d_sigma, m->d_flag, n, m->t.err, ctx->rank, W);
    CU(ctx, cudaGetLastError());
  }
  // Ordering of the return sections.  Owners store into rank r's return section only between barrier 1 (in send) and
  // barrier 2 (below) of a call; rank r reads it after barrier 2, and enqueues that read before its own barrier 1 of the
  // next call.  coll_barrier is stream-ordered (an NCCL all-reduce on the stream, or a stream synchronise and then the
  // host barrier on a loopback world), so no owner's next stores can overtake the read: no second region set and no
  // third barrier are needed.
  st = m->x.done(ctx, s);
  if (st != BW_OK) return st;
  if (refuse != BW_OK) CTX_FAIL(ctx, refuse, "%s", why);
  if (refused >= 0) CTX_FAIL(ctx, BW_ERR_STATE, "smap: rank %d refused this call (its own error says why); no rank mapped it", refused);
  const XchgRet ret = m->x.ret_mine();
  if (rows) {
    const cudaMemcpyKind kind = host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    CU(ctx, cudaMemcpyAsync(mu, ret.mu, rows * 8, kind, s));
    CU(ctx, cudaMemcpyAsync(sigma, ret.sigma, rows * 8, kind, s));
    CU(ctx, cudaMemcpyAsync(flag, ret.flag, rows, kind, s));
  }
  CU(ctx, cudaMemcpyAsync(m->h_ret_err, ret.err, W * sizeof(u32), cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  int full = -1;
  for (int r = W - 1; r >= 0; --r)
    if (m->h_ret_err[r]) full = r;
  if (full >= 0) {
    m->failed = true;
    const u32 e = m->h_ret_err[ctx->rank];
    if (e) CTX_FAIL(ctx, (bw_status)e, "smap kernel raised status %u: key table full (raise capacity_hint)", e);
    CTX_FAIL(ctx, BW_ERR_STATE, "smap: rank %d's key table is full; this call's results are invalid and the map is unusable", full);
  }
  return BW_OK;
}

bw_status bw_smap_apply_device(bw_smap* m, const uint64_t* d_keys, const void* d_vals, uint64_t rows, double* d_mu,
                               double* d_sigma, uint8_t* d_flag) {
  if (!m) return BW_ERR_SPEC;
  bw_ctx* ctx = m->ctx;
  if (m->shard) return smap_apply_ranks(m, d_keys, d_vals, rows, d_mu, d_sigma, d_flag, false);
  if (rows > m->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "smap: rows > max_batch_rows");
  if (rows == 0) return BW_OK;
  CU(ctx, cudaSetDevice(ctx->device));
  return smap_map(m, d_keys, d_vals, rows, d_mu, d_sigma, d_flag);
}

bw_status bw_smap_sync(bw_smap* m) {
  if (!m) return BW_ERR_SPEC;
  bw_ctx* ctx = m->ctx;
  CU(ctx, cudaMemcpyAsync(m->h_err, m->t.err, 4, cudaMemcpyDeviceToHost, m->s));
  CU(ctx, cudaStreamSynchronize(m->s));
  if (*m->h_err) CTX_FAIL(ctx, (bw_status)*m->h_err, "smap kernel raised status %u: key table full (raise capacity_hint)", *m->h_err);
  if (m->failed) CTX_FAIL(ctx, BW_ERR_STATE, "smap: an earlier call failed; the map is unusable");
  return BW_OK;
}

bw_status bw_smap_apply(bw_smap* m, const uint64_t* keys, const void* vals, uint64_t rows, double* out_mu, double* out_sigma,
                        uint8_t* out_flag) {
  if (!m) return BW_ERR_SPEC;
  bw_ctx* ctx = m->ctx;
  if (m->shard) return smap_apply_ranks(m, keys, vals, rows, out_mu, out_sigma, out_flag, true);
  if (rows > m->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "smap: rows > max_batch_rows");
  if (rows == 0) return BW_OK;
  CU(ctx, cudaSetDevice(ctx->device));
  const size_t vb = m->spec.val_dtype == BW_VAL_F32 ? 4 : 8;
  CU(ctx, cudaMemcpyAsync(m->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, m->s));
  CU(ctx, cudaMemcpyAsync(m->d_vals, vals, rows * vb, cudaMemcpyHostToDevice, m->s));
  bw_status st = bw_smap_apply_device(m, m->k.d_keys, m->d_vals, rows, m->d_mu, m->d_sigma, m->d_flag);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(out_mu, m->d_mu, rows * 8, cudaMemcpyDeviceToHost, m->s));
  CU(ctx, cudaMemcpyAsync(out_sigma, m->d_sigma, rows * 8, cudaMemcpyDeviceToHost, m->s));
  CU(ctx, cudaMemcpyAsync(out_flag, m->d_flag, rows, cudaMemcpyDeviceToHost, m->s));
  return bw_smap_sync(m);
}

struct bw_join {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_join_spec spec{};
  JoinSlot* slots = nullptr;
  u64 cap = 0;
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32 *d_err = nullptr, *h_err = nullptr;
  unsigned long long *d_nrows = nullptr, *h_nrows = nullptr;
  unsigned char* d_side = nullptr;
  u64* d_vals = nullptr;
  JoinEmit e{};
  SortScratch srt;  // ordering scratch
  HostCols h;       // host output: key, left, right, mask, epoch
  u32 batch_no = 0;
  u64 min_epoch = 0, last_epoch = 0;
  bool pending = false;
  // world > 1: the exchange, and the source columns it sends
  RankXchg x;
  u64 *d_src_keys = nullptr, *d_src_vals = nullptr;
  unsigned char* d_src_side = nullptr;
  i64* d_src_side64 = nullptr;
};

// Source buffers and the exchange of a join on world > 1 (collective): the side rides in the 8-byte ts column.
static bw_status join_ranks_setup(bw_join* j) {
  bw_ctx* ctx = j->ctx;
  Owner& own = j->own;
  const u64 B = j->spec.max_batch_rows;
  CU(ctx, own.dev(&j->d_src_keys, B));
  CU(ctx, own.dev(&j->d_src_vals, B));
  CU(ctx, own.dev(&j->d_src_side, B));
  CU(ctx, own.dev(&j->d_src_side64, B));
  return j->x.setup(ctx, own, B, false, false, 0, j->s);
}

bw_status bw_join_create(bw_ctx* ctx, const bw_join_spec* spec, bw_join** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_join_create: NULL argument");
  if (spec->struct_size != sizeof(bw_join_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_join_spec.struct_size mismatch");
  if (spec->insert_mode < 0 || spec->insert_mode > 1) CTX_FAIL(ctx, BW_ERR_SPEC, "insert_mode must be first or last (product: host path)");
  if (spec->emit_mode < 0 || spec->emit_mode > 2) CTX_FAIL(ctx, BW_ERR_SPEC, "bad emit_mode");
  // an owner groups up to max_batch_rows from every rank with 32-bit sort indices and sequence numbers
  if (spec->max_batch_rows == 0 || spec->max_batch_rows > ((1ULL << 31) - 1) / (u64)ctx->world)
    CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows: max_batch_rows * world must be in [1, 2^31)");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_join, void (*)(bw_join*)> jp(new bw_join(), bw_join_destroy);  // torn down on every failure
  bw_join* j = jp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  j->cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&j->slots, j->cap + 1));
  CU(ctx, own.dev(&j->d_err, 1));
  CU(ctx, own.dev(&j->d_nrows, 1));
  CU(ctx, cudaMemsetAsync(j->d_err, 0, 4, j->s));
  CU(ctx, cudaMemsetAsync(j->d_nrows, 0, 8, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_nrows, 64 / sizeof(unsigned long long)));
  // rows one activation brings to this rank: its own on one GPU, up to max_batch_rows from every rank on world > 1
  const u64 n = spec->max_batch_rows * (u64)ctx->world, m = std::max<u64>(spec->max_emit_rows, 1024);
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_side, n));
  CU(ctx, own.dev(&j->d_vals, n));
  for (u64** c : {&j->e.key, &j->e.l, &j->e.r, &j->e.mask, &j->e.seq, &j->e.epoch}) CU(ctx, own.dev(c, m));
  j->e.max_rows = spec->max_emit_rows;
  j->e.n_rows = j->d_nrows;
  CU(ctx, j->srt.reserve(own, m, m, j->s));
  CU(ctx, j->h.reserve(own, m, m));
  k_join_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(j->slots, j->cap);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  if (ctx->world > 1) {
    st = join_ranks_setup(j);
    if (st != BW_OK) return st;
  }
  *out = jp.release();
  return BW_OK;
}

void bw_join_destroy(bw_join* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  j->x.close(j->ctx);
  delete j;  // j->own releases every buffer and the stream
}

// bw_join_apply on world > 1 (include/bwgpu.h): every row to its key's owner, then K6 there over what arrived.
static bw_status join_apply_ranks(bw_join* j, const u64* keys, const uint8_t* side, const u64* vals, u64 rows, u64 epoch) {
  bw_ctx* ctx = j->ctx;
  const int W = ctx->world;
  cudaStream_t s = j->s;
  CU(ctx, cudaSetDevice(ctx->device));
  // A call that cannot go ahead still takes part in the exchange and both barriers, so that no peer waits for it in a
  // barrier: it sends no rows and raises its refusal flag, and every rank then fails the call.
  bw_status refuse = BW_OK;
  const char* why = "";
  if (rows > j->spec.max_batch_rows) {
    refuse = BW_ERR_SPEC;
    why = "join: rows > max_batch_rows";
  } else if (rows && (!keys || !side || !vals)) {
    refuse = BW_ERR_SPEC;
    why = "join: NULL column";
  } else if (j->pending && epoch < j->last_epoch) {
    refuse = BW_ERR_STATE;
    why = "join: epochs must not decrease";
  }
  if (refuse != BW_OK) rows = 0;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(j->d_src_keys, keys, rows * 8, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(j->d_src_side, side, rows, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(j->d_src_vals, vals, rows * 8, cudaMemcpyHostToDevice, s));
  }
  PartIn in;
  in.keys = j->d_src_keys;
  in.vals = j->d_src_vals;
  in.ts = j->d_src_side64;
  in.n = rows;
  in.val_bytes = 8;
  in.world = W;
  const int grid = (int)std::min<u64>(std::max<u64>((rows + BW_PART_TILE - 1) / BW_PART_TILE, 1), (u64)ctx->sm_count * 8);
  k_xjoin_side<<<grid, BW_PART_THREADS, 0, s>>>(j->d_src_side, j->d_src_side64, rows);
  // K6 has no clock: the head's time row carries 0
  bw_status st = j->x.send(ctx, s, in, epoch, 0, refuse != BW_OK);
  if (st != BW_OK) return st;
  // every rank reads the same head: all of them fail here, or none does
  const u64 *got_epoch = j->x.head(1), *got_refused = j->x.head(3);
  int refused = -1, epoch_differs = -1;
  for (int r = W - 1; r >= 0; --r) {
    if (got_refused[r]) refused = r;
    if (got_epoch[r] != got_epoch[0]) epoch_differs = r;
  }
  const bool go = refused < 0 && epoch_differs < 0;
  u64 n = 0;
  if (go) {
    BatchView bv;
    n = j->x.received(ctx, bv);
    if (n) k_xjoin_gather<<<ctx->sm_count * 4, 256, 0, s>>>(bv, n, j->k.d_keys, j->d_vals, j->d_side);
    CU(ctx, cudaGetLastError());
  }
  // barrier 2 on every call, failed or not: past it no peer's next call stores into this region or its head before
  // this rank has read them
  st = j->x.done(ctx, s);
  if (st != BW_OK) return st;
  if (refuse != BW_OK) CTX_FAIL(ctx, refuse, "%s", why);
  if (refused >= 0) CTX_FAIL(ctx, BW_ERR_STATE, "join: rank %d refused this call (its own error says why); no rank played it", refused);
  if (epoch_differs >= 0)
    CTX_FAIL(ctx, BW_ERR_STATE, "join: rank 0 played epoch %llu and rank %d epoch %llu; every rank must pass the same epoch to one call",
             (unsigned long long)got_epoch[0], epoch_differs, (unsigned long long)got_epoch[epoch_differs]);
  if (!j->pending) {
    j->min_epoch = epoch;
    j->pending = true;
  }
  j->last_epoch = epoch;
  const u32 batch_no = j->batch_no++;
  if (n) {
    st = keyed_group(ctx, j->k, j->k.d_keys, n, s);
    if (st != BW_OK) return st;
    k_join_apply<<<ctx->sm_count * 8, 256, 0, s>>>(j->slots, j->cap, j->d_err, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, j->d_side,
                                                    j->d_vals, n, j->spec.insert_mode, j->spec.emit_mode, j->e, batch_no, epoch);
    CU(ctx, cudaGetLastError());
  }
  CU(ctx, cudaStreamSynchronize(s));
  return BW_OK;
}

bw_status bw_join_apply(bw_join* j, const uint64_t* keys, const uint8_t* side, const uint64_t* vals, uint64_t rows, uint64_t epoch) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  if (ctx->world > 1) return join_apply_ranks(j, keys, side, vals, rows, epoch);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "join: rows > max_batch_rows");
  if (j->pending && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "join: epochs must not decrease");
  if (!j->pending) {
    j->min_epoch = epoch;
    j->pending = true;
  }
  j->last_epoch = epoch;
  const u32 batch_no = j->batch_no++;
  if (rows == 0) return BW_OK;
  CU(ctx, cudaSetDevice(ctx->device));
  CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, j->s));
  CU(ctx, cudaMemcpyAsync(j->d_side, side, rows, cudaMemcpyHostToDevice, j->s));
  CU(ctx, cudaMemcpyAsync(j->d_vals, vals, rows * 8, cudaMemcpyHostToDevice, j->s));
  bw_status st = keyed_group(ctx, j->k, j->k.d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_join_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->slots, j->cap, j->d_err, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, j->d_side,
                                                      j->d_vals, rows, j->spec.insert_mode, j->spec.emit_mode, j->e, batch_no, epoch);
  CU(ctx, cudaGetLastError());
  // the host columns may be reused by the caller once this returns
  CU(ctx, cudaStreamSynchronize(j->s));
  return BW_OK;
}

static bw_status join_collect(bw_join* j, bw_join_rows* out) {
  bw_ctx* ctx = j->ctx;
  cudaStream_t s = j->s;
  CU(ctx, cudaMemcpyAsync(j->h_err, j->d_err, 4, cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaMemcpyAsync(j->h_nrows, j->d_nrows, 8, cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  if (*j->h_err) CTX_FAIL(ctx, (bw_status)*j->h_err, "join kernel raised status %u: key table or emit buffer full", *j->h_err);
  const u64 n = std::min<u64>(*j->h_nrows, j->e.max_rows);
  if (n) {
    SortScratch& x = j->srt;
    bw_status st = order_perm(ctx, x, s, n, j->e.key, j->e.seq, j->e.epoch, nullptr, j->last_epoch - j->min_epoch + 1, j->min_epoch,
                              nullptr);
    if (st != BW_OK) return st;
    const u64* src[] = {j->e.key, j->e.l, j->e.r, j->e.mask, j->e.epoch};
    for (int c = 0; c < 5; ++c) {
      k_gather_u64<<<ctx->sm_count * 4, 256, 0, s>>>(src[c], x.perm, x.gather, n);
      CU(ctx, cudaMemcpyAsync(j->h.col[c], x.gather, n * 8, cudaMemcpyDeviceToHost, s));
    }
    CU(ctx, cudaGetLastError());
  }
  CU(ctx, cudaMemsetAsync(j->d_nrows, 0, 8, s));
  CU(ctx, cudaStreamSynchronize(s));
  j->pending = false;
  out->n = n;
  out->key = j->h.col[0];
  out->left = j->h.col[1];
  out->right = j->h.col[2];
  out->mask = j->h.col[3];
  out->epoch = j->h.col[4];
  return BW_OK;
}

bw_status bw_join_advance(bw_join* j, bw_join_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  CU(j->ctx, cudaSetDevice(j->ctx->device));
  return join_collect(j, out);
}

bw_status bw_join_eof(bw_join* j, bw_join_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (!j->pending) {
    j->min_epoch = j->last_epoch;
    j->pending = true;
  }
  k_join_eof<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->slots, j->cap, j->d_err, j->spec.emit_mode, j->e, j->last_epoch);
  CU(ctx, cudaGetLastError());
  return join_collect(j, out);
}

// ===========================================================================
// K7 host side: session-window folds (bw_session.cuh)
// ===========================================================================
struct bw_session {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_session_spec spec{};
  SessTable t{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;                    // err, why
  unsigned long long* d_cnt = nullptr;     // closed rows, merged ids, late rows
  unsigned long long* h_cnt = nullptr;
  u64* d_vals = nullptr;
  i64* d_ts = nullptr;
  SessEmit e{};
  SortScratch srt;  // ordering scratch
  HostCols hc[2];   // closed: key, window id, acc, open, close | epoch, merged count, merged offset
  HostCols hl;      // late: key, epoch, activation, row, source rank
  i64* h_mids = nullptr;
  std::vector<u64> merged_off;
  std::vector<i64> merged_ids;
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
  // world > 1: the exchange (with source rows), each gathered row's name (source rank << 32 | source row), and the late
  // row count before a fold
  RankXchg x;
  u64* d_name = nullptr;
  unsigned long long* d_late0 = nullptr;
};

bw_status bw_session_create(bw_ctx* ctx, const bw_session_spec* user, bw_session** out) {
  if (!ctx || !user || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_session_create: NULL argument");
  // a spec built against the header before shard_by_key existed ends just before it, and leaves it 0
  if (user->struct_size != sizeof(bw_session_spec) && user->struct_size != offsetof(bw_session_spec, shard_by_key))
    CTX_FAIL(ctx, BW_ERR_SPEC, "bw_session_spec.struct_size mismatch");
  bw_session_spec copy{};
  memcpy(&copy, user, user->struct_size);
  const bw_session_spec* spec = &copy;
  if (ctx->world != 1 && !spec->shard_by_key)
    CTX_FAIL(ctx, BW_ERR_SPEC, "session folds run on one GPU (world == 1) unless the spec sets shard_by_key");
  if (spec->reduction < BW_RED_COUNT || spec->reduction > BW_RED_MAX) CTX_FAIL(ctx, BW_ERR_SPEC, "reduction must be count, sum, min or max");
  if (spec->val_dtype != BW_VAL_I64 && spec->val_dtype != BW_VAL_F64) CTX_FAIL(ctx, BW_ERR_SPEC, "val_dtype must be I64 or F64");
  if (spec->gap_us < 0 || spec->gap_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "gap_us must be in 0..UTC_MAX - UTC_MIN");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_sessions_per_key < 1 || spec->max_sessions_per_key > BW_SESS_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_sessions_per_key must be in 1..%d", BW_SESS_MAXM);
  // an owner groups up to max_batch_rows from every rank with 32-bit sort indices
  if (spec->max_batch_rows == 0 || spec->max_batch_rows > ((1ULL << 31) - 1) / (u64)ctx->world)
    CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows: max_batch_rows * world must be in [1, 2^31)");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_session, void (*)(bw_session*)> sp(new bw_session(), bw_session_destroy);  // torn down on every failure
  bw_session* f = sp.get();
  Owner& own = f->own;
  f->ctx = ctx;
  f->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_sessions_per_key;
  SessTable& t = f->t;
  t.cap = cap;
  t.M = M;
  CU(ctx, own.stream(&f->s));
  CU(ctx, own.dev(&t.keys, cap + 1));
  CU(ctx, own.dev(&t.st, cap + 1));
  CU(ctx, own.dev(&t.rec, (cap + 1) * (u64)M));
  CU(ctx, own.dev(&t.mrg, (cap + 1) * (u64)(2 * M)));
  CU(ctx, own.dev(&t.err, 2));
  t.why = t.err + 1;
  CU(ctx, own.dev(&f->d_cnt, 3));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, f->s));
  CU(ctx, cudaMemsetAsync(f->d_cnt, 0, 24, f->s));
  CU(ctx, own.host(&f->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&f->h_cnt, 64 / sizeof(unsigned long long)));
  // rows one activation brings to this rank: its own on one GPU, up to max_batch_rows from every rank on world > 1
  const u64 n = spec->max_batch_rows * (u64)ctx->world, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  bw_status st = keyed_alloc(ctx, own, f->k, n, f->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&f->d_vals, n));
  CU(ctx, own.dev(&f->d_ts, n));
  SessEmit& e = f->e;
  for (u64** c : {&e.key, &e.acc, &e.epoch, &e.ord, &e.moff, &e.mcnt}) CU(ctx, own.dev(c, m));
  for (i64** c : {&e.wid, &e.open, &e.close, &e.mids}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_epoch, &e.l_ord, &e.l_act, &e.l_row}) CU(ctx, own.dev(c, l));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.n_rows = f->d_cnt;
  e.n_mids = f->d_cnt + 1;
  e.n_late = f->d_cnt + 2;
  CU(ctx, f->srt.reserve(own, std::max(m, l), std::max(m, l), f->s));
  CU(ctx, f->hc[0].reserve(own, m, m));
  CU(ctx, f->hc[1].reserve(own, m, m));
  CU(ctx, f->hl.reserve(own, l, l));
  CU(ctx, own.host(&f->h_mids, m));
  k_session_init<<<ctx->sm_count * 4, 256, 0, f->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(f->s));
  if (ctx->world > 1) {
    CU(ctx, own.dev(&f->d_name, n));
    CU(ctx, own.dev(&f->d_late0, 1));
    st = f->x.setup(ctx, own, spec->max_batch_rows, true, false, 0, f->s);
    if (st != BW_OK) return st;
  }
  *out = sp.release();
  return BW_OK;
}

void bw_session_destroy(bw_session* f) {
  if (!f) return;
  cudaSetDevice(f->ctx->device);
  if (f->s) cudaStreamSynchronize(f->s);
  f->x.close(f->ctx);
  delete f;  // f->own releases every buffer and the stream
}

static SessParams session_params(bw_session* f, u64 epoch) {
  SessParams p;
  p.red = f->spec.reduction;
  p.is_f64 = f->spec.val_dtype == BW_VAL_F64;
  p.gap = f->spec.gap_us;
  p.wait = f->spec.wait_us;
  p.now = f->now;
  p.epoch = epoch;
  p.ord = f->calls++;
  p.batch_no = f->batch_no;
  return p;
}

// `now_getter()` of the call: never goes backwards (windowing.py:250-261)
static void session_now(bw_session* f, int64_t system_now_us) {
  if (system_now_us > f->now) f->now = system_now_us;
}

static bw_status session_check(bw_session* f) {
  bw_ctx* ctx = f->ctx;
  if (f->failed) CTX_FAIL(ctx, BW_ERR_STATE, "session fold: an earlier call ran out of capacity; the fold is unusable");
  CU(ctx, cudaMemcpyAsync(f->h_err, f->t.err, 8, cudaMemcpyDeviceToHost, f->s));
  CU(ctx, cudaStreamSynchronize(f->s));
  if (f->h_err[0]) {
    f->failed = true;
    const u32 w = f->h_err[1];
    CTX_FAIL(ctx, (bw_status)f->h_err[0], "session kernel ran out of capacity:%s%s%s%s%s", w & BW_SESS_FULL_TABLE ? " key table full (raise capacity_hint);" : "",
             w & BW_SESS_FULL_SESSIONS ? " a key needs more than max_sessions_per_key sessions or merged ids;" : "",
             w & BW_SESS_FULL_EMIT ? " more than max_emit_rows closed sessions or merged ids since the last advance;" : "",
             w & BW_SESS_FULL_LATE ? " more than max_late_rows late rows since the last advance;" : "", w ? "" : " (no reason recorded)");
  }
  return BW_OK;
}

// bw_session_apply / _apply_device on world > 1 (include/bwgpu.h): every row to its key's owner, then K7 there over what
// arrived.  `host`: the columns are host memory.
static bw_status session_apply_ranks(bw_session* f, const u64* keys, const void* vals, const i64* ts_us, u64 rows, u64 epoch,
                                     i64 system_now_us, bool host) {
  bw_ctx* ctx = f->ctx;
  const int W = ctx->world;
  const bool count = f->spec.reduction == BW_RED_COUNT;
  cudaStream_t s = f->s;
  CU(ctx, cudaSetDevice(ctx->device));
  // A call that cannot go ahead still takes part in the exchange and both barriers, so that no peer waits for it in a
  // barrier: it sends no rows and raises its refusal flag, and every rank then fails the call.
  bw_status refuse = BW_OK;
  std::string why;
  if (f->failed) {
    refuse = BW_ERR_STATE;
    why = "session fold: an earlier call ran out of capacity; the fold is unusable";
  } else if (rows > f->spec.max_batch_rows) {
    refuse = BW_ERR_SPEC;
    why = "session: rows > max_batch_rows";
  } else if (rows && (!keys || !ts_us || (!vals && !count))) {
    refuse = BW_ERR_SPEC;
    why = "session: NULL column";
  } else if (f->batch_no && epoch < f->last_epoch) {
    refuse = BW_ERR_STATE;
    why = "session: epochs must not decrease";
  } else if ((refuse = session_check(f)) != BW_OK) {  // a full table or session list met by an earlier apply_device
    why = ctx->err;
  }
  if (refuse != BW_OK) rows = 0;
  PartIn in;
  in.keys = keys;
  in.vals = count ? nullptr : vals;
  in.ts = ts_us;
  in.n = rows;
  in.val_bytes = count ? 0 : 8;
  in.world = W;
  if (host && rows) {  // staged in K7's own columns: the gather overwrites them only after the scatter has read them
    CU(ctx, cudaMemcpyAsync(f->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(f->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, s));
    if (!count) CU(ctx, cudaMemcpyAsync(f->d_vals, vals, rows * 8, cudaMemcpyHostToDevice, s));
    in.keys = f->k.d_keys;
    in.vals = count ? nullptr : f->d_vals;
    in.ts = f->d_ts;
  }
  bw_status st = f->x.send(ctx, s, in, epoch, system_now_us, refuse != BW_OK);
  if (st != BW_OK) return st;
  // every rank reads the same head: all of them fail here, or none does
  const u64 *got_epoch = f->x.head(1), *got_now = f->x.head(2), *got_refused = f->x.head(3);
  int refused = -1, epoch_differs = -1, now_differs = -1;
  for (int r = W - 1; r >= 0; --r) {
    if (got_refused[r]) refused = r;
    if (got_epoch[r] != got_epoch[0]) epoch_differs = r;
    if (got_now[r] != got_now[0]) now_differs = r;
  }
  const bool go = refused < 0 && epoch_differs < 0 && now_differs < 0;
  u64 n = 0;
  if (go) {
    BatchView bv;
    n = f->x.received(ctx, bv);
    if (n)
      k_xsess_gather<<<ctx->sm_count * 4, 256, 0, s>>>(bv, f->x.rows(), f->spec.max_batch_rows, n, f->k.d_keys, count ? nullptr : f->d_vals,
                                                       f->d_ts, f->d_name);
    CU(ctx, cudaGetLastError());
  }
  st = f->x.done(ctx, s);
  if (st != BW_OK) return st;
  if (refuse != BW_OK) CTX_FAIL(ctx, refuse, "%s", why.c_str());
  if (refused >= 0) CTX_FAIL(ctx, BW_ERR_STATE, "session: rank %d refused this call (its own error says why); no rank folded it", refused);
  if (epoch_differs >= 0)
    CTX_FAIL(ctx, BW_ERR_STATE, "session: rank 0 played epoch %llu and rank %d epoch %llu; every rank must pass the same epoch to one call",
             (unsigned long long)got_epoch[0], epoch_differs, (unsigned long long)got_epoch[epoch_differs]);
  if (now_differs >= 0)
    CTX_FAIL(ctx, BW_ERR_STATE,
             "session: rank 0 passed system_now_us %lld and rank %d %lld; every rank must pass the same system time to one call",
             (long long)got_now[0], now_differs, (long long)got_now[now_differs]);
  f->last_epoch = epoch;
  session_now(f, system_now_us);
  const SessParams p = session_params(f, epoch);
  f->batch_no++;
  if (n) {
    st = keyed_group(ctx, f->k, f->k.d_keys, n, s);
    if (st != BW_OK) return st;
    CU(ctx, cudaMemcpyAsync(f->d_late0, f->e.n_late, 8, cudaMemcpyDeviceToDevice, s));
    k_session_apply<<<ctx->sm_count * 8, 256, 0, s>>>(f->t, f->e, p, f->k.d_ksorted, f->k.d_isorted, f->k.d_head,
                                                      count ? nullptr : f->d_vals, f->d_ts, n);
    k_xsess_name_late<<<ctx->sm_count * 4, 256, 0, s>>>(f->d_late0, f->e.n_late, f->e.max_late, f->e.l_row, f->d_name);
    CU(ctx, cudaGetLastError());
  }
  return host ? session_check(f) : BW_OK;
}

bw_status bw_session_apply_device(bw_session* f, const uint64_t* d_keys, const void* d_vals, const int64_t* d_ts_us, uint64_t rows,
                                  uint64_t epoch, int64_t system_now_us) {
  if (!f) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (ctx->world > 1) return session_apply_ranks(f, d_keys, d_vals, d_ts_us, rows, epoch, system_now_us, false);
  if (f->failed) CTX_FAIL(ctx, BW_ERR_STATE, "session fold: an earlier call ran out of capacity; the fold is unusable");
  if (rows > f->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "session: rows > max_batch_rows");
  if (rows && (!d_keys || !d_ts_us || (!d_vals && f->spec.reduction != BW_RED_COUNT))) CTX_FAIL(ctx, BW_ERR_SPEC, "session: NULL column");
  if (f->batch_no && epoch < f->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "session: epochs must not decrease");
  f->last_epoch = epoch;
  session_now(f, system_now_us);
  CU(ctx, cudaSetDevice(ctx->device));
  const SessParams p = session_params(f, epoch);
  f->batch_no++;
  if (rows == 0) return BW_OK;
  bw_status st = keyed_group(ctx, f->k, d_keys, rows, f->s);
  if (st != BW_OK) return st;
  k_session_apply<<<ctx->sm_count * 8, 256, 0, f->s>>>(f->t, f->e, p, f->k.d_ksorted, f->k.d_isorted, f->k.d_head, (const u64*)d_vals,
                                                       d_ts_us, rows);
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

bw_status bw_session_apply(bw_session* f, const uint64_t* keys, const void* vals, const int64_t* ts_us, uint64_t rows, uint64_t epoch,
                           int64_t system_now_us) {
  if (!f) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (ctx->world > 1) return session_apply_ranks(f, keys, vals, ts_us, rows, epoch, system_now_us, true);
  if (rows > f->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "session: rows > max_batch_rows");
  CU(ctx, cudaSetDevice(ctx->device));
  const bool has_vals = vals != nullptr;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(f->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, f->s));
    CU(ctx, cudaMemcpyAsync(f->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, f->s));
    if (has_vals) CU(ctx, cudaMemcpyAsync(f->d_vals, vals, rows * 8, cudaMemcpyHostToDevice, f->s));
  }
  bw_status st = bw_session_apply_device(f, f->k.d_keys, has_vals ? f->d_vals : nullptr, f->d_ts, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return session_check(f);
}

static bw_status session_collect(bw_session* f, bw_session_rows* out) {
  bw_ctx* ctx = f->ctx;
  cudaStream_t s = f->s;
  bw_status st = session_check(f);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(f->h_cnt, f->d_cnt, 24, cudaMemcpyDeviceToHost, s));
  CU(ctx, cudaStreamSynchronize(s));
  const u64 nc = f->h_cnt[0], nmid = f->h_cnt[1], nl = f->h_cnt[2];  // all within bounds: session_check passed
  const u64 n_ord = std::max<u64>(f->calls - f->first_call, 1);
  const int grid = ctx->sm_count * 4;
  SortScratch& x = f->srt;
  const SessEmit& e = f->e;
  if (nc) {  // per call, key string, then session id (the id column doubles as the sequence)
    st = order_perm(ctx, x, s, nc, e.key, (const u64*)e.wid, e.ord, nullptr, n_ord, f->first_call, nullptr);
    if (st != BW_OK) return st;
    const u64* src[] = {e.key, (const u64*)e.wid, e.acc, (const u64*)e.open, (const u64*)e.close, e.epoch, e.mcnt, e.moff};
    for (int c = 0; c < 8; ++c) {
      k_gather_u64<<<grid, 256, 0, s>>>(src[c], x.perm, x.gather, nc);
      CU(ctx, cudaMemcpyAsync(f->hc[c / 5].col[c % 5], x.gather, nc * 8, cudaMemcpyDeviceToHost, s));
    }
    if (nmid) CU(ctx, cudaMemcpyAsync(f->h_mids, e.mids, nmid * 8, cudaMemcpyDeviceToHost, s));
  }
  if (nl) {  // per call, key string, then arrival order (the row column holds names: source rank << 32 | source row)
    st = order_perm(ctx, x, s, nl, e.l_key, e.l_row, e.l_ord, nullptr, n_ord, f->first_call, nullptr);
    if (st != BW_OK) return st;
    const u64* src[] = {e.l_key, e.l_epoch, e.l_act, e.l_row};
    for (int c = 0; c < 4; ++c) {
      k_gather_u64<<<grid, 256, 0, s>>>(src[c], x.perm, x.gather, nl);
      CU(ctx, cudaMemcpyAsync(f->hl.col[c], x.gather, nl * 8, cudaMemcpyDeviceToHost, s));
    }
  }
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(f->d_cnt, 0, 24, s));
  CU(ctx, cudaStreamSynchronize(s));
  u64 *lrow = f->hl.col[3], *lrank = f->hl.col[4];
  for (u64 i = 0; i < nl; ++i) {
    lrank[i] = lrow[i] >> 32;
    lrow[i] &= 0xffffffffULL;
  }
  // merged ids in row order
  f->merged_off.assign(nc + 1, 0);
  f->merged_ids.resize(nmid);
  const u64 *cnt = f->hc[1].col[1], *off = f->hc[1].col[2];
  for (u64 r = 0; r < nc; ++r) {
    f->merged_off[r + 1] = f->merged_off[r] + cnt[r];
    std::copy(f->h_mids + off[r], f->h_mids + off[r] + cnt[r], f->merged_ids.begin() + f->merged_off[r]);
  }
  f->first_call = f->calls;
  out->n_closed = nc;
  out->closed_key = f->hc[0].col[0];
  out->closed_window_id = (const int64_t*)f->hc[0].col[1];
  out->closed_acc = f->hc[0].col[2];
  out->closed_open_us = (const int64_t*)f->hc[0].col[3];
  out->closed_close_us = (const int64_t*)f->hc[0].col[4];
  out->closed_epoch = f->hc[1].col[0];
  out->merged_off = f->merged_off.data();
  out->merged_ids = f->merged_ids.data();
  out->n_late = nl;
  out->late_key = f->hl.col[0];
  out->late_epoch = f->hl.col[1];
  out->late_activation = f->hl.col[2];
  out->late_row = f->hl.col[3];
  out->late_rank = f->hl.col[4];
  return BW_OK;
}

bw_status bw_session_advance(bw_session* f, int64_t system_now_us, bw_session_rows* out) {
  if (!f || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (f->failed) CTX_FAIL(ctx, BW_ERR_STATE, "session fold: an earlier call ran out of capacity; the fold is unusable");
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    session_now(f, system_now_us);
    k_session_close_all<<<ctx->sm_count * 8, 256, 0, f->s>>>(f->t, f->e, session_params(f, f->last_epoch), 0);
    CU(ctx, cudaGetLastError());
  }
  return session_collect(f, out);
}

bw_status bw_session_eof(bw_session* f, bw_session_rows* out) {
  if (!f || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = f->ctx;
  if (f->failed) CTX_FAIL(ctx, BW_ERR_STATE, "session fold: an earlier call ran out of capacity; the fold is unusable");
  CU(ctx, cudaSetDevice(ctx->device));
  k_session_close_all<<<ctx->sm_count * 8, 256, 0, f->s>>>(f->t, f->e, session_params(f, f->last_epoch), 1);
  CU(ctx, cudaGetLastError());
  return session_collect(f, out);
}

// ===========================================================================
// K8 host side: windowed join (bw_jwin.cuh)
// ===========================================================================
struct bw_jwin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_jwin_spec spec{};
  JwTable t{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;                 // err, why
  unsigned long long* d_cnt = nullptr;  // down, meta, late, released, carried-over queue entries
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_side = nullptr, *d_late = nullptr;
  u64* d_handles = nullptr;
  i64* d_ts = nullptr;
  JwEmit e{};
  JwPool pool{}, pool2{};  // ordered mode: the queue, and the one the next flush writes
  u64 nq = 0;              // entries in `pool`
  int slot_bits = 1;
  SortScratch srt;       // pool sort and ordering scratch
  HostCols hd[2];        // down: key, window id, h0, h1, h2 | h3, mask, epoch
  HostCols hm, hl;       // meta: key, window id, epoch; late: key, window id, epoch, activation, row
  std::vector<u64> late_rank;     // the late rows' source ranks, split off their row column
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;     // a call whose released handles and queue count are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
  // world > 1: the exchange (with source rows and sides), each gathered row's name (source rank << 32 | source row),
  // and the late row count before a call
  RankXchg x;
  u64* d_name = nullptr;
  unsigned long long* d_late0 = nullptr;
};

static bw_status jwin_pool_alloc(bw_ctx* ctx, Owner& own, JwPool& p, u64 n) {
  CU(ctx, own.dev(&p.slot, n));
  CU(ctx, own.dev(&p.ts, n));
  CU(ctx, own.dev(&p.h, n));
  CU(ctx, own.dev(&p.side, n));
  return BW_OK;
}

bw_status bw_jwin_create(bw_ctx* ctx, const bw_jwin_spec* user, bw_jwin** out) {
  if (!ctx || !user || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_jwin_create: NULL argument");
  // a spec built against the header before shard_by_key existed ends just before it, and leaves it 0
  if (user->struct_size != sizeof(bw_jwin_spec) && user->struct_size != offsetof(bw_jwin_spec, shard_by_key))
    CTX_FAIL(ctx, BW_ERR_SPEC, "bw_jwin_spec.struct_size mismatch");
  bw_jwin_spec copy{};
  memcpy(&copy, user, user->struct_size);
  const bw_jwin_spec* spec = &copy;
  if (ctx->world != 1 && !spec->shard_by_key)
    CTX_FAIL(ctx, BW_ERR_SPEC, "windowed joins run on one GPU (world == 1) unless the spec sets shard_by_key");
  if (spec->insert_mode != BW_JOIN_INSERT_FIRST && spec->insert_mode != BW_JOIN_INSERT_LAST)
    CTX_FAIL(ctx, BW_ERR_SPEC, "insert_mode must be first or last (product: host engine)");
  if (spec->emit_mode < BW_JOIN_EMIT_COMPLETE || spec->emit_mode > BW_JOIN_EMIT_RUNNING) CTX_FAIL(ctx, BW_ERR_SPEC, "bad emit_mode");
  if (spec->ordered != 0 && spec->ordered != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "ordered must be 0 or 1");
  if (spec->sides < 1 || spec->sides > BW_JW_MAXSIDES) CTX_FAIL(ctx, BW_ERR_SPEC, "sides must be in 1..%d", BW_JW_MAXSIDES);
  if (spec->max_windows_per_key < 1 || spec->max_windows_per_key > BW_JW_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_windows_per_key must be in 1..%d", BW_JW_MAXM);
  if (spec->length_us <= 0 || spec->length_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "length_us must be in 1..UTC_MAX - UTC_MIN");
  if (spec->offset_us <= 0 || spec->offset_us > spec->length_us) CTX_FAIL(ctx, BW_ERR_SPEC, "offset_us must be in 1..length_us");
  if (spec->align_us < BW_UTC_MIN_US || spec->align_us > BW_UTC_MAX_US) CTX_FAIL(ctx, BW_ERR_SPEC, "align_us out of range");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  // an owner groups and sorts up to max_batch_rows from every rank, and its pool, with 32-bit indices
  if (spec->max_batch_rows == 0 || spec->max_batch_rows > ((1ULL << 31) - 1) / (u64)ctx->world)
    CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows: max_batch_rows * world must be in [1, 2^31)");
  if (spec->max_queued_rows >= (1ULL << 31) - spec->max_batch_rows * (u64)ctx->world)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_queued_rows + max_batch_rows * world must stay below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_jwin, void (*)(bw_jwin*)> jp(new bw_jwin(), bw_jwin_destroy);  // torn down on every failure
  bw_jwin* j = jp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_windows_per_key;
  JwTable& t = j->t;
  t.cap = cap;
  t.M = M;
  t.sides = spec->sides;
  while ((1ULL << j->slot_bits) < cap + 1) ++j->slot_bits;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.keys, cap + 1));
  CU(ctx, own.dev(&t.st, cap + 1));
  CU(ctx, own.dev(&t.win, (cap + 1) * (u64)M));
  CU(ctx, own.dev(&t.err, 2));
  t.why = t.err + 1;
  CU(ctx, own.dev(&j->d_cnt, 5));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 40, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 64 / sizeof(unsigned long long)));
  // rows one activation brings to this rank: its own on one GPU, up to max_batch_rows from every rank on world > 1
  const u64 n = spec->max_batch_rows * (u64)ctx->world, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  const u64 q = spec->ordered ? spec->max_queued_rows : 0;
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_side, n));
  CU(ctx, own.dev(&j->d_late, n));
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_ts, n));
  if (spec->ordered) {
    if ((st = jwin_pool_alloc(ctx, own, j->pool, q + n)) != BW_OK) return st;
    if ((st = jwin_pool_alloc(ctx, own, j->pool2, q + n)) != BW_OK) return st;
  }
  JwEmit& e = j->e;
  for (u64** c : {&e.key, &e.wid, &e.h0, &e.h1, &e.h2, &e.h3, &e.mask, &e.epoch, &e.ord, &e.seq}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.m_key, &e.m_wid, &e.m_epoch, &e.m_ord, &e.m_seq}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  // the release buffer grows with the handles held (jwin_room); it starts at one batch
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.max_queue = q;
  e.n_rows = j->d_cnt;
  e.n_meta = j->d_cnt + 1;
  e.n_late = j->d_cnt + 2;
  e.n_rel = j->d_cnt + 3;
  e.n_next = j->d_cnt + 4;
  const u64 ns = std::max(std::max(m, l), q + n);
  CU(ctx, j->srt.reserve(own, ns, ns, j->s));
  CU(ctx, j->hd[0].reserve(own, m, m));
  CU(ctx, j->hd[1].reserve(own, m, m));
  CU(ctx, j->hm.reserve(own, m, m));
  CU(ctx, j->hl.reserve(own, l, l));
  k_jwin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  if (ctx->world > 1) {
    CU(ctx, own.dev(&j->d_name, n));
    CU(ctx, own.dev(&j->d_late0, 1));
    st = j->x.setup(ctx, own, spec->max_batch_rows, true, true, 0, j->s);
    if (st != BW_OK) return st;
  }
  *out = jp.release();
  return BW_OK;
}

void bw_jwin_destroy(bw_jwin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  j->x.close(j->ctx);
  delete j;  // j->own releases every buffer and the stream
}

static JwParams jwin_params(bw_jwin* j, u64 epoch) {
  JwParams p;
  p.insert_last = j->spec.insert_mode == BW_JOIN_INSERT_LAST;
  p.emit_mode = j->spec.emit_mode;
  p.ordered = j->spec.ordered;
  p.length = j->spec.length_us;
  p.offset = j->spec.offset_us;
  p.align = j->spec.align_us;
  p.wait = j->spec.wait_us;
  p.now = j->now;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.batch_no = j->batch_no;
  return p;
}

#define JWIN_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "windowed join: an earlier call failed on the device; the join is unusable")

// What differs between the handle joins that share the host steps below (J: bw_jwin, K8; bw_sjwin, K10, whose overloads
// follow its struct): the name in messages, what BW_JW_FULL_WINDOWS / BW_JW_FULL_EMIT mean, the device counters.
static const char* jwin_what(const bw_jwin*) { return "windowed join"; }
static const char* jwin_full_windows(const bw_jwin*) { return " a key needs more than max_windows_per_key open windows;"; }
static const char* jwin_full_emit(const bw_jwin*) { return " more than max_emit_rows down or meta rows since the last advance;"; }
static u64 jwin_counters(const bw_jwin*) { return 5; }  // down, meta, late, released, carried-over queue entries
// ordered joins keep a queue whose entry count comes back with the drain (bw_argwin, K11, has none)
template <class J>
static bool jwin_queues(const J* j) {
  return j->spec.ordered;
}

// wait for the last call; fail on a device-side overflow; then take its released handles and its queue count, so the
// device buffer only ever holds one call's releases
template <class J>
static bw_status jwin_drain(J* j) {
  bw_ctx* ctx = j->ctx;
  if (j->failed) CTX_FAIL(ctx, BW_ERR_STATE, "%s: an earlier call failed on the device; the join is unusable", jwin_what(j));
  if (!j->undrained) return BW_OK;
  CU(ctx, cudaMemcpyAsync(j->h_err, j->t.err, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 8 * jwin_counters(j), cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  if (j->h_err[0]) {
    j->failed = true;
    const u32 w = j->h_err[1];
    CTX_FAIL(ctx, (bw_status)j->h_err[0], "%s kernel %s:%s%s%s%s%s%s%s%s%s", jwin_what(j),
             j->h_err[0] == BW_ERR_SPEC ? "rejected its input" : "ran out of capacity",
             w & BW_JW_BAD_SIDE ? " a side column value is not below sides;" : "", w & BW_JW_FULL_TABLE ? " key table full (raise capacity_hint);" : "",
             w & BW_JW_FULL_WINDOWS ? jwin_full_windows(j) : "",
             w & BW_JW_FULL_EMIT ? jwin_full_emit(j) : "",
             w & BW_JW_FULL_LATE ? " more than max_late_rows late rows since the last advance;" : "",
             w & BW_JW_FULL_QUEUE ? " more than max_queued_rows queued entries;" : "",
             w & BW_CW_FULL_STORE ? " entry store or staging buffer full;" : "",
             w & BW_PJ_FULL_SIDE ? " a window's side list reached 2^32 values;" : "", w ? "" : " (no reason recorded)");
  }
  const u64 nr = j->h_cnt[3];
  j->outstanding -= std::min(nr, j->outstanding);
  if (nr) {
    const size_t at = j->released.size();
    j->released.resize(at + nr);
    CU(ctx, cudaMemcpyAsync(j->released.data() + at, j->e.rel, nr * 8, cudaMemcpyDeviceToHost, j->s));
  }
  if (jwin_queues(j)) j->nq = j->h_cnt[4];
  CU(ctx, cudaMemsetAsync(j->d_cnt + 3, 0, 16, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->undrained = false;
  return BW_OK;
}

// Room in the release buffer for the next call: it can release at most the handles passed in earlier and not released
// yet, plus its own `rows`.  Called after jwin_drain, so nothing on the stream reads the old buffer and it holds no
// releases; the buffer then holds what the join actually holds, not what its tables could hold.  (J: bw_jwin, bw_collect)
template <class J>
static bw_status jwin_room(J* j, u64 rows) {
  const u64 need = j->outstanding + rows;
  if (need <= j->e.max_rel) return BW_OK;
  const u64 grow = std::max<u64>(need, 2 * j->e.max_rel);
  j->e.max_rel = 0;  // (a failed regrow leaves no buffer: the next call tries again)
  CU(j->ctx, j->own.regrow(Owner::DEV, &j->e.rel, grow));
  j->e.max_rel = grow;
  return BW_OK;
}

// ordered mode: put the n entries of `pool` in play order -- x.perm: every key's due entries by ts (ties in arrival
// order), then the rest in arrival order, keys by slot -- and give every key its range (k_jwin_ranges).  (J: bw_jwin,
// bw_collect)
template <class J>
static bw_status jwin_sort_pool(J* j, const JwTable& t, const JwParams& p, u64 n) {
  bw_ctx* ctx = j->ctx;
  const int grid = ctx->sm_count * 4;
  SortScratch& x = j->srt;
  if (!n) return BW_OK;
  k_jwin_sortkey<<<grid, 256, 0, j->s>>>(t, p, j->pool, x.sk, x.perm, n);
  size_t tb = x.cub_bytes;
  CU(ctx, cub::DeviceRadixSort::SortPairs(x.cub, tb, x.sk, x.sk2, x.perm, x.perm2, (int)n, 0, 64, j->s));
  k_jwin_slotkey<<<grid, 256, 0, j->s>>>(j->pool, x.perm2, x.sk, n);
  tb = x.cub_bytes;
  CU(ctx, cub::DeviceRadixSort::SortPairs(x.cub, tb, x.sk, x.sk2, x.perm2, x.perm, (int)n, 0, j->slot_bits, j->s));
  k_jwin_ranges<<<grid, 256, 0, j->s>>>(t, p, j->pool, x.perm, n);
  return BW_OK;
}

// ordered mode: sort the pool's due entries into play order, then flush every woken key: `flush(e, perm)` launches the
// join's flush kernel (k_jwin_flush, k_sjwin_flush) with emit buffers whose carry-over pool is the next one
template <class J, class F>
static bw_status jwin_flush_pool(J* j, const JwParams& p, u64 n, F&& flush) {
  bw_ctx* ctx = j->ctx;
  bw_status st = jwin_sort_pool(j, j->t, p, n);
  if (st != BW_OK) return st;
  auto e = j->e;
  e.next = j->pool2;
  flush(e, j->srt.perm);
  CU(ctx, cudaGetLastError());
  std::swap(j->pool, j->pool2);  // the next call reads what this flush carried over (count: jwin_drain)
  return BW_OK;
}
static bw_status jwin_flush_pool(bw_jwin* j, const JwParams& p, u64 n) {
  return jwin_flush_pool(j, p, n, [&](const JwEmit& e, const u32* perm) {
    k_jwin_flush<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, p, j->pool, perm);
  });
}

// bw_jwin_apply / _apply_device on world > 1 (include/bwgpu.h): every row to its key's owner, then K8 there over what
// arrived.  `host`: the columns are host memory.
static bw_status jwin_apply_ranks(bw_jwin* j, const u64* keys, const uint8_t* side, const u64* handles, const i64* ts_us, u64 rows,
                                  u64 epoch, i64 system_now_us, bool host) {
  bw_ctx* ctx = j->ctx;
  const int W = ctx->world;
  cudaStream_t s = j->s;
  CU(ctx, cudaSetDevice(ctx->device));
  // A call that cannot go ahead still takes part in the exchange and both barriers, so that no peer waits for it in a
  // barrier: it sends no rows and raises its refusal flag, and every rank then fails the call.
  bw_status refuse = BW_OK;
  std::string why;
  if (j->failed) {
    refuse = BW_ERR_STATE;
    why = "windowed join: an earlier call failed on the device; the join is unusable";
  } else if (rows > j->spec.max_batch_rows) {
    refuse = BW_ERR_SPEC;
    why = "windowed join: rows > max_batch_rows";
  } else if (rows && (!keys || !side || !handles || !ts_us)) {
    refuse = BW_ERR_SPEC;
    why = "windowed join: NULL column";
  } else if (j->batch_no && epoch < j->last_epoch) {
    refuse = BW_ERR_STATE;
    why = "windowed join: epochs must not decrease";
  } else if ((refuse = jwin_drain(j)) != BW_OK) {  // a device error met by an earlier apply_device
    why = ctx->err;
  }
  for (u64 i = 0; host && refuse == BW_OK && i < rows; ++i)
    if (side[i] >= (u32)j->spec.sides) {
      refuse = BW_ERR_SPEC;
      why = "windowed join: side " + std::to_string(side[i]) + " of row " + std::to_string(i) + " is not below sides";
    }
  if (refuse != BW_OK) rows = 0;
  PartIn in;
  in.keys = keys;
  in.vals = handles;
  in.ts = ts_us;
  in.n = rows;
  in.val_bytes = 8;
  in.world = W;
  const unsigned char* in_side = side;
  if (host && rows) {  // staged in K8's own columns: the gather overwrites them only after the scatter has read them
    CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(j->d_side, side, rows, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(j->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, s));
    CU(ctx, cudaMemcpyAsync(j->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, s));
    in.keys = j->k.d_keys;
    in.vals = j->d_handles;
    in.ts = j->d_ts;
    in_side = j->d_side;
  }
  bw_status st = j->x.send(ctx, s, in, epoch, system_now_us, refuse != BW_OK, in_side);
  if (st != BW_OK) return st;
  // every rank reads the same head: all of them fail here, or none does
  const u64 *got_epoch = j->x.head(1), *got_now = j->x.head(2), *got_refused = j->x.head(3);
  int refused = -1, epoch_differs = -1, now_differs = -1;
  for (int r = W - 1; r >= 0; --r) {
    if (got_refused[r]) refused = r;
    if (got_epoch[r] != got_epoch[0]) epoch_differs = r;
    if (got_now[r] != got_now[0]) now_differs = r;
  }
  const bool go = refused < 0 && epoch_differs < 0 && now_differs < 0;
  u64 n = 0;
  if (go) {
    BatchView bv;
    n = j->x.received(ctx, bv);
    if (n)
      k_xjwin_gather<<<ctx->sm_count * 4, 256, 0, s>>>(bv, j->x.rows(), j->x.side(), j->spec.max_batch_rows, n, j->k.d_keys, j->d_handles,
                                                       j->d_side, j->d_ts, j->d_name);
    CU(ctx, cudaGetLastError());
  }
  st = j->x.done(ctx, s);
  if (st != BW_OK) return st;
  if (refuse != BW_OK) CTX_FAIL(ctx, refuse, "%s", why.c_str());
  if (refused >= 0) CTX_FAIL(ctx, BW_ERR_STATE, "windowed join: rank %d refused this call (its own error says why); no rank played it", refused);
  if (epoch_differs >= 0)
    CTX_FAIL(ctx, BW_ERR_STATE,
             "windowed join: rank 0 played epoch %llu and rank %d epoch %llu; every rank must pass the same epoch to one call",
             (unsigned long long)got_epoch[0], epoch_differs, (unsigned long long)got_epoch[epoch_differs]);
  if (now_differs >= 0)
    CTX_FAIL(ctx, BW_ERR_STATE,
             "windowed join: rank 0 passed system_now_us %lld and rank %d %lld; every rank must pass the same system time to one call",
             (long long)got_now[0], now_differs, (long long)got_now[now_differs]);
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = jwin_params(j, epoch);
  j->batch_no++;
  if (n) {
    // the n rows received (not max_batch_rows x W): the release buffer holds what the join holds
    if ((st = jwin_room(j, n)) != BW_OK) return st;
    j->outstanding += n;
    st = keyed_group(ctx, j->k, j->k.d_keys, n, s);
    if (st != BW_OK) return st;
    CU(ctx, cudaMemcpyAsync(j->d_late0, j->e.n_late, 8, cudaMemcpyDeviceToDevice, s));
    k_jwin_apply<<<ctx->sm_count * 8, 256, 0, s>>>(j->t, j->e, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, j->d_handles,
                                                   j->d_side, j->d_ts, j->d_late, n);
    k_xjwin_name_late<<<ctx->sm_count * 4, 256, 0, s>>>(j->d_late0, j->e.n_late, j->e.max_late, j->e.l_row, j->d_name, n);
    CU(ctx, cudaGetLastError());
    j->undrained = true;
    if (j->spec.ordered && (st = jwin_flush_pool(j, p, j->nq + n)) != BW_OK) return st;
  }
  // the host columns may be reused by the caller once this returns
  return host ? jwin_drain(j) : BW_OK;
}

bw_status bw_jwin_apply_device(bw_jwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles, const int64_t* d_ts_us,
                               uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  if (ctx->world > 1) return jwin_apply_ranks(j, d_keys, d_side, d_handles, d_ts_us, rows, epoch, system_now_us, false);
  JWIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed join: rows > max_batch_rows");
  if (rows && (!d_keys || !d_side || !d_handles || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed join: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "windowed join: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = jwin_params(j, epoch);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = jwin_room(j, rows)) != BW_OK) return st;
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_jwin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, d_handles,
                                                    d_side, d_ts_us, j->d_late, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return jwin_flush_pool(j, p, j->nq + rows);
  return BW_OK;
}

// one activation from HOST columns: check the sides, copy the columns to the join's device columns, run `apply_device`,
// and wait, so the caller may reuse its columns (J: bw_jwin, bw_sjwin)
template <class J, class D>
static bw_status jwin_apply_host(J* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us, uint64_t rows,
                                 uint64_t epoch, int64_t system_now_us, D apply_device) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "%s: rows > max_batch_rows", jwin_what(j));
  if (rows && (!keys || !side || !handles || !ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "%s: NULL column", jwin_what(j));
  for (u64 i = 0; i < rows; ++i)
    if (side[i] >= (u32)j->spec.sides)
      CTX_FAIL(ctx, BW_ERR_SPEC, "%s: side %u of row %llu is not below sides", jwin_what(j), side[i], (unsigned long long)i);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_side, side, rows, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, j->s));
  }
  st = apply_device(j, j->k.d_keys, j->d_side, j->d_handles, j->d_ts, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return jwin_drain(j);
}

bw_status bw_jwin_apply(bw_jwin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us, uint64_t rows,
                        uint64_t epoch, int64_t system_now_us) {
  if (j && j->ctx->world > 1) return jwin_apply_ranks(j, keys, side, handles, ts_us, rows, epoch, system_now_us, true);
  return jwin_apply_host(j, keys, side, handles, ts_us, rows, epoch, system_now_us, bw_jwin_apply_device);
}

// order rows [0, n) of one stream by (call, key string, seq) and copy `nc` columns to the host (J: bw_jwin, bw_collect)
template <class J>
static bw_status jwin_ship(J* j, u64 n, const u64* key, const u64* seq, const u64* ord, const u64* const* src, int nc, HostCols* dst) {
  if (!n) return BW_OK;
  bw_ctx* ctx = j->ctx;
  SortScratch& x = j->srt;
  bw_status st = order_perm(ctx, x, j->s, n, key, seq, ord, nullptr, std::max<u64>(j->calls - j->first_call, 1), j->first_call, nullptr);
  if (st != BW_OK) return st;
  for (int c = 0; c < nc; ++c) {
    k_gather_u64<<<ctx->sm_count * 4, 256, 0, j->s>>>(src[c], x.perm, x.gather, n);
    CU(ctx, cudaMemcpyAsync(dst[c / 5].col[c % 5], x.gather, n * 8, cudaMemcpyDeviceToHost, j->s));
  }
  return BW_OK;
}

static bw_status jwin_collect(bw_jwin* j, bw_jwin_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 24, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 nd = j->h_cnt[0], nm = j->h_cnt[1], nl = j->h_cnt[2];  // all within bounds: jwin_drain passed
  const JwEmit& e = j->e;
  const u64* down[] = {e.key, e.wid, e.h0, e.h1, e.h2, e.h3, e.mask, e.epoch};
  const u64* meta[] = {e.m_key, e.m_wid, e.m_epoch};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(j, nd, e.key, e.seq, e.ord, down, 8, j->hd)) != BW_OK) return st;
  if ((st = jwin_ship(j, nm, e.m_key, e.m_seq, e.m_ord, meta, 3, &j->hm)) != BW_OK) return st;
  if ((st = jwin_ship(j, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &j->hl)) != BW_OK) return st;
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 24, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  // the row column holds names, source rank << 32 | source row (on world 1 the rank is 0)
  u64* lrow = j->hl.col[4];
  j->late_rank.resize(nl);
  for (u64 i = 0; i < nl; ++i) {
    j->late_rank[i] = lrow[i] >> 32;
    lrow[i] &= 0xffffffffULL;
  }
  j->first_call = j->calls;
  out->n_down = nd;
  out->down_key = j->hd[0].col[0];
  out->down_window_id = (const int64_t*)j->hd[0].col[1];
  out->down_handle[0] = j->hd[0].col[2];
  out->down_handle[1] = j->hd[0].col[3];
  out->down_handle[2] = j->hd[0].col[4];
  out->down_handle[3] = j->hd[1].col[0];
  out->down_mask = j->hd[1].col[1];
  out->down_epoch = j->hd[1].col[2];
  out->n_meta = nm;
  out->meta_key = j->hm.col[0];
  out->meta_window_id = (const int64_t*)j->hm.col[1];
  out->meta_epoch = j->hm.col[2];
  out->n_late = nl;
  out->late_key = j->hl.col[0];
  out->late_window_id = (const int64_t*)j->hl.col[1];
  out->late_epoch = j->hl.col[2];
  out->late_activation = j->hl.col[3];
  out->late_row = j->hl.col[4];
  out->late_rank = j->late_rank.data();
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys, then flush them (ordered: through the pool)
static bw_status jwin_wake(bw_jwin* j, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  if ((st = jwin_room(j, 0)) != BW_OK) return st;
  const JwParams p = jwin_params(j, j->last_epoch);
  k_jwin_mark<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->t.win, p, eof);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return jwin_flush_pool(j, p, j->nq);
  JwEmit e = j->e;
  k_jwin_flush<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, p, j->pool, nullptr);
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

bw_status bw_jwin_advance(bw_jwin* j, int64_t system_now_us, bw_jwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  JWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > j->now) j->now = system_now_us;
    bw_status st = jwin_wake(j, 0);
    if (st != BW_OK) return st;
  }
  return jwin_collect(j, out);
}

bw_status bw_jwin_eof(bw_jwin* j, bw_jwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  JWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = jwin_wake(j, 1);
  if (st != BW_OK) return st;
  return jwin_collect(j, out);
}

// ===========================================================================
// K9 host side: collect_window (bw_collect.cuh)
// ===========================================================================
struct bw_collect {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_collect_spec spec{};
  CwTable t{};
  CwStore es{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;                 // err, why
  unsigned long long* d_cnt = nullptr;  // closed windows, late rows, released, carried-over queue entries, staged, store
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_late = nullptr, *d_flag = nullptr;
  u64* d_handles = nullptr;
  i64* d_ts = nullptr;
  CwEmit e{};
  JwPool pool{}, pool2{};  // ordered mode: the queue, and the one the next flush writes
  u64 nq = 0;              // entries in `pool`
  int slot_bits = 1;
  u64 kmax = 1;            // entries one value can add: min(ceil(length / offset), max_windows_per_key)
  u64 n_store = 0, dead = 0;      // entries in the store, and how many of them are dead
  u64 n_rows = 0, n_stage = 0;    // closed windows and staged handles since the last advance / eof
  SortScratch srt;                // pool sort, ordering and compaction scratch
  u32* d_inv = nullptr;           // advance / eof: a closed window's place in the reference's order
  u64 *d_cs = nullptr, *d_off = nullptr;  // its count in that order, and the exclusive scan of them
  u64* d_out = nullptr;           // the handles in the reference's order
  u64* h_out = nullptr;
  u64 out_cap = 0;
  HostCols hd, hl;                // down: key, window id, epoch, offsets; late: key, window id, epoch, activation, row
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;     // a call whose counts are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
};

bw_status bw_collect_create(bw_ctx* ctx, const bw_collect_spec* spec, bw_collect** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_collect_create: NULL argument");
  if (spec->struct_size != sizeof(bw_collect_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_collect_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed collects run on one GPU (world == 1)");
  if (spec->ordered != 0 && spec->ordered != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "ordered must be 0 or 1");
  if (spec->max_windows_per_key < 1 || spec->max_windows_per_key > BW_JW_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_windows_per_key must be in 1..%d", BW_JW_MAXM);
  if (spec->length_us <= 0 || spec->length_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "length_us must be in 1..UTC_MAX - UTC_MIN");
  if (spec->offset_us <= 0 || spec->offset_us > spec->length_us) CTX_FAIL(ctx, BW_ERR_SPEC, "offset_us must be in 1..length_us");
  if (spec->align_us < BW_UTC_MIN_US || spec->align_us > BW_UTC_MAX_US) CTX_FAIL(ctx, BW_ERR_SPEC, "align_us out of range");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_queued_rows >= (1ULL << 31) - spec->max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "max_queued_rows + max_batch_rows must stay below 2^31");
  if (spec->max_emit_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "max_emit_rows must be below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_collect, void (*)(bw_collect*)> cp(new bw_collect(), bw_collect_destroy);  // torn down on every failure
  bw_collect* j = cp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_windows_per_key;
  const u64 per = (u64)((spec->length_us - 1) / spec->offset_us) + 1;
  j->kmax = std::min<u64>(per, (u64)M);
  CwTable& t = j->t;
  t.j.cap = cap;
  t.j.M = M;
  t.j.sides = 1;
  while ((1ULL << j->slot_bits) < cap + 1) ++j->slot_bits;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.j.keys, cap + 1));
  CU(ctx, own.dev(&t.j.st, cap + 1));
  CU(ctx, own.dev(&t.win, (cap + 1) * (u64)M));
  CU(ctx, own.dev(&t.cell_ord, (cap + 1) * (u64)M));
  CU(ctx, own.dev(&t.cell_c, (cap + 1) * (u64)M));
  CU(ctx, own.dev(&t.j.err, 2));
  t.j.why = t.j.err + 1;
  t.err = t.j.err;
  t.why = t.j.why;
  CU(ctx, own.dev(&j->d_cnt, 6));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 48, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 64 / sizeof(unsigned long long)));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  const u64 q = spec->ordered ? spec->max_queued_rows : 0;
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_late, n));
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_ts, n));
  if (spec->ordered) {
    if ((st = jwin_pool_alloc(ctx, own, j->pool, q + n)) != BW_OK) return st;
    if ((st = jwin_pool_alloc(ctx, own, j->pool2, q + n)) != BW_OK) return st;
  }
  CwEmit& e = j->e;
  for (u64** c : {&e.key, &e.wid, &e.cnt, &e.soff, &e.epoch, &e.ord, &e.seq}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  CU(ctx, own.dev(&j->d_inv, m));
  CU(ctx, own.dev(&j->d_cs, m + 1));
  CU(ctx, own.dev(&j->d_off, m + 1));
  // the store, the staging buffer, the output and the release buffer grow with what the collect holds (collect_room);
  // they start at one batch
  CwStore& es = j->es;
  es.cap = n;
  CU(ctx, own.dev(&es.ref, n));
  CU(ctx, own.dev(&es.rank, n));
  CU(ctx, own.dev(&es.h, n));
  CU(ctx, own.dev(&j->d_flag, n));
  e.max_stage = n;
  CU(ctx, own.dev(&e.stage, n));
  CU(ctx, own.dev(&e.stage_rec, n));
  j->out_cap = n;
  CU(ctx, own.dev(&j->d_out, n));
  CU(ctx, own.host(&j->h_out, n));
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.max_queue = q;
  e.n_rows = j->d_cnt;
  e.n_late = j->d_cnt + 1;
  e.n_rel = j->d_cnt + 2;
  e.n_next = j->d_cnt + 3;
  e.n_stage = j->d_cnt + 4;
  es.n = j->d_cnt + 5;
  const u64 ns = std::max(std::max(m, l), q + n);
  CU(ctx, j->srt.reserve(own, ns, ns, j->s));
  size_t b = 0;
  CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b, j->d_cs, j->d_off, (int)(m + 1), j->s));
  CU(ctx, j->srt.grow_cub(own, b + 256));
  CU(ctx, j->hd.reserve(own, m + 1, m + 1));
  CU(ctx, j->hl.reserve(own, l, l));
  k_cwin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = cp.release();
  return BW_OK;
}

void bw_collect_destroy(bw_collect* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static JwParams collect_params(bw_collect* j, u64 epoch) {
  JwParams p{};
  p.ordered = j->spec.ordered;
  p.length = j->spec.length_us;
  p.offset = j->spec.offset_us;
  p.align = j->spec.align_us;
  p.wait = j->spec.wait_us;
  p.now = j->now;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.batch_no = j->batch_no;
  return p;
}

#define COLLECT_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "windowed collect: an earlier call failed on the device; the collect is unusable")

// wait for the last call; fail on a device-side overflow; then take its released handles and its counts
static bw_status collect_drain(bw_collect* j) {
  bw_ctx* ctx = j->ctx;
  COLLECT_REFUSE_FAILED(j);
  if (!j->undrained) return BW_OK;
  CU(ctx, cudaMemcpyAsync(j->h_err, j->t.err, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 48, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  if (j->h_err[0]) {
    j->failed = true;
    const u32 w = j->h_err[1];
    CTX_FAIL(ctx, (bw_status)j->h_err[0], "windowed collect kernel ran out of capacity:%s%s%s%s%s%s%s",
             w & BW_JW_FULL_TABLE ? " key table full (raise capacity_hint);" : "",
             w & BW_JW_FULL_WINDOWS ? " a key needs more than max_windows_per_key open windows;" : "",
             w & BW_JW_FULL_EMIT ? " more than max_emit_rows closed windows since the last advance;" : "",
             w & BW_JW_FULL_LATE ? " more than max_late_rows late rows since the last advance;" : "",
             w & BW_JW_FULL_QUEUE ? " more than max_queued_rows queued entries;" : "",
             w & BW_CW_FULL_STORE ? " entry store or staging buffer full;" : "", w ? "" : " (no reason recorded)");
  }
  const u64 nr = j->h_cnt[2];
  j->outstanding -= std::min(nr, j->outstanding);
  if (nr) {
    const size_t at = j->released.size();
    j->released.resize(at + nr);
    CU(ctx, cudaMemcpyAsync(j->released.data() + at, j->e.rel, nr * 8, cudaMemcpyDeviceToHost, j->s));
  }
  if (j->spec.ordered) j->nq = j->h_cnt[3];
  j->n_rows = j->h_cnt[0];
  j->dead += j->h_cnt[4] - j->n_stage;  // every staged handle left a dead entry behind
  j->n_stage = j->h_cnt[4];
  j->n_store = j->h_cnt[5];
  CU(ctx, cudaMemsetAsync(j->d_cnt + 2, 0, 16, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->undrained = false;
  return BW_OK;
}

// a device buffer of `cap` elements, the first `used` of them kept, regrown to `grow` (nothing on the stream reads it)
// (J: bw_collect, bw_scwin)
template <class J, class T>
static cudaError_t collect_grow_keep(J* j, T** p, u64 used, u64 grow) {
  T* q = nullptr;
  cudaError_t e = j->own.dev(&q, grow);
  if (!e && used) e = cudaMemcpyAsync(q, *p, used * sizeof(T), cudaMemcpyDeviceToDevice, j->s);
  if (!e) e = cudaStreamSynchronize(j->s);
  if (e) {
    j->own.release(q);
    return e;
  }
  j->own.release(*p);
  *p = q;
  return cudaSuccess;
}

// emit buffers whose staging buffer has a record column (K9, K12, K13; K15 stages by rank ranges and has none)
template <class E, class = void>
struct HasStageRec : std::false_type {};
template <class E>
struct HasStageRec<E, std::void_t<decltype(&E::stage_rec)>> : std::true_type {};

// Before a call that can add `adds` entries to the store: compact the store once dead entries outnumber live ones, then
// grow the store and the staging buffer so that nothing the call can add or stage overflows them.  Called after the
// drain: nothing on the stream reads them.  (J: bw_collect, bw_scwin, bw_kcollect, bw_kjoin)
template <class J>
static bw_status store_room(J* j, u64 adds) {
  bw_ctx* ctx = j->ctx;
  auto& es = j->es;
  auto& e = j->e;
  if (j->dead && j->dead >= j->n_store - j->dead) {  // stream compaction (entry order does not matter: each has its rank)
    const int grid = ctx->sm_count * 4;
    k_cwin_live<<<grid, 256, 0, j->s>>>(es.ref, j->d_flag, j->n_store);
    size_t b = 0;
    CU(ctx, cub::DeviceSelect::Flagged(nullptr, b, es.ref, j->d_flag, es.n, (int64_t)j->n_store, j->s));
    CU(ctx, j->srt.grow_cub(j->own, b + 256));
    for (int c = 0; c < 3; ++c) {
      size_t tb = j->srt.cub_bytes;
      if (c == 0) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.h, j->d_flag, es.n, (int64_t)j->n_store, j->s));
      if (c == 1) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.rank, j->d_flag, es.n, (int64_t)j->n_store, j->s));
      if (c == 2) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.ref, j->d_flag, es.n, (int64_t)j->n_store, j->s));
    }
    CU(ctx, cudaGetLastError());
    j->n_store -= j->dead;
    j->dead = 0;
  }
  const u64 live = j->n_store - j->dead;
  if (j->n_store + adds > es.cap) {
    const u64 grow = std::max<u64>(j->n_store + adds, 2 * es.cap);
    es.cap = 0;  // (a failed regrow leaves the store unusable: the next call fails here again)
    CU(ctx, collect_grow_keep(j, &es.ref, j->n_store, grow));
    CU(ctx, collect_grow_keep(j, &es.rank, j->n_store, grow));
    CU(ctx, collect_grow_keep(j, &es.h, j->n_store, grow));
    CU(ctx, j->own.regrow(Owner::DEV, &j->d_flag, grow));
    es.cap = grow;
  }
  if (j->n_stage + live + adds > e.max_stage) {
    const u64 grow = std::max<u64>(j->n_stage + live + adds, 2 * e.max_stage);
    e.max_stage = 0;
    CU(ctx, collect_grow_keep(j, &e.stage, j->n_stage, grow));
    if constexpr (HasStageRec<std::decay_t<decltype(e)>>::value) CU(ctx, collect_grow_keep(j, &e.stage_rec, j->n_stage, grow));
    e.max_stage = grow;
  }
  return BW_OK;
}

// Before a call that can play `rows` values (and ordered the queued entries): room in the store, the staging buffer and
// the release buffer for all it can add or close.  (J: bw_collect, bw_scwin)
template <class J>
static bw_status collect_room(J* j, u64 rows) {
  bw_status st = jwin_room(j, rows);
  if (st != BW_OK) return st;
  return store_room(j, (rows + (j->spec.ordered ? j->nq : 0)) * j->kmax);
}

// after the per-key kernels of a call: move the closed windows' entries out (k_cwin_gather)
static bw_status collect_gather(bw_collect* j, const JwParams& p) {
  k_cwin_gather<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->n_rows);
  CU(j->ctx, cudaGetLastError());
  return BW_OK;
}

// ordered mode: sort the pool's due entries into play order (K8's sort), then flush every woken key (k_cwin_flush)
static bw_status collect_flush(bw_collect* j, const JwParams& p, u64 n) {
  bw_ctx* ctx = j->ctx;
  bw_status st = j->spec.ordered ? jwin_sort_pool(j, j->t.j, p, n) : BW_OK;
  if (st != BW_OK) return st;
  CwEmit e = j->e;
  e.next = j->pool2;
  k_cwin_flush<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, j->es, p, j->pool, j->srt.perm);
  CU(ctx, cudaGetLastError());
  if (j->spec.ordered) std::swap(j->pool, j->pool2);  // the next call reads what this flush carried over (count: collect_drain)
  return collect_gather(j, p);
}

bw_status bw_collect_apply_device(bw_collect* j, const uint64_t* d_keys, const uint64_t* d_handles, const int64_t* d_ts_us, uint64_t rows,
                                  uint64_t epoch, int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  COLLECT_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed collect: rows > max_batch_rows");
  if (rows && (!d_keys || !d_handles || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed collect: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "windowed collect: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = collect_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = collect_params(j, epoch);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = collect_room(j, rows)) != BW_OK) return st;
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_cwin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted, j->k.d_head,
                                                    d_handles, d_ts_us, j->d_late, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return collect_flush(j, p, j->nq + rows);
  return collect_gather(j, p);
}

bw_status bw_collect_apply(bw_collect* j, const uint64_t* keys, const uint64_t* handles, const int64_t* ts_us, uint64_t rows, uint64_t epoch,
                           int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed collect: rows > max_batch_rows");
  if (rows && (!keys || !handles || !ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed collect: NULL column");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = collect_drain(j);
  if (st != BW_OK) return st;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, j->s));
  }
  st = bw_collect_apply_device(j, j->k.d_keys, j->d_handles, j->d_ts, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return collect_drain(j);
}

// advance / eof, after jwin_ship put the nd closed records in the reference's order (x.perm): their lists as CSR --
// offsets (nd + 1 of them, to h_off) by a scan of their counts, then every one of the ns staged handles to its place in
// parallel, to h_out (J: bw_collect, bw_scwin)
template <class J>
static bw_status collect_place(J* j, u64 nd, u64 ns, u64* h_off) {
  bw_ctx* ctx = j->ctx;
  if (ns > j->out_cap) {
    j->out_cap = 0;
    CU(ctx, j->own.regrow(Owner::DEV, &j->d_out, ns));
    CU(ctx, j->own.regrow(Owner::HOST, &j->h_out, ns));
    j->out_cap = ns;
  }
  if (!nd) {
    h_off[0] = 0;
    return BW_OK;
  }
  const int grid = ctx->sm_count * 4;
  SortScratch& x = j->srt;
  const auto& e = j->e;
  k_cwin_order<<<grid, 256, 0, j->s>>>(x.perm, e.cnt, j->d_inv, j->d_cs, nd);
  CU(ctx, cudaMemsetAsync(j->d_cs + nd, 0, 8, j->s));
  size_t tb = x.cub_bytes;
  CU(ctx, cub::DeviceScan::ExclusiveSum(x.cub, tb, j->d_cs, j->d_off, (int)(nd + 1), j->s));
  k_cwin_place<<<ctx->sm_count * 8, 256, 0, j->s>>>(e.stage, e.stage_rec, e.soff, j->d_inv, j->d_off, j->d_out, ns);
  CU(ctx, cudaMemcpyAsync(h_off, j->d_off, (nd + 1) * 8, cudaMemcpyDeviceToHost, j->s));
  if (ns) CU(ctx, cudaMemcpyAsync(j->h_out, j->d_out, ns * 8, cudaMemcpyDeviceToHost, j->s));
  return BW_OK;
}

static bw_status collect_collect(bw_collect* j, bw_collect_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = collect_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 48, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 nd = j->h_cnt[0], nl = j->h_cnt[1], ns = j->h_cnt[4];  // all within bounds: collect_drain passed
  const CwEmit& e = j->e;
  const u64* down[] = {e.key, e.wid, e.epoch};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(j, nd, e.key, e.seq, e.ord, down, 3, &j->hd)) != BW_OK) return st;
  if ((st = collect_place(j, nd, ns, j->hd.col[3])) != BW_OK) return st;
  if ((st = jwin_ship(j, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &j->hl)) != BW_OK) return st;
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 16, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 4, 0, 8, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->n_rows = j->n_stage = 0;
  j->first_call = j->calls;
  out->n_down = nd;
  out->down_key = j->hd.col[0];
  out->down_window_id = (const int64_t*)j->hd.col[1];
  out->down_epoch = j->hd.col[2];
  out->down_offset = j->hd.col[3];
  out->handle = j->h_out;
  out->n_late = nl;
  out->late_key = j->hl.col[0];
  out->late_window_id = (const int64_t*)j->hl.col[1];
  out->late_epoch = j->hl.col[2];
  out->late_activation = j->hl.col[3];
  out->late_row = j->hl.col[4];
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys (K8's k_jwin_mark), then flush them (ordered: through the pool)
static bw_status collect_wake(bw_collect* j, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = collect_drain(j);
  if (st != BW_OK) return st;
  if ((st = collect_room(j, 0)) != BW_OK) return st;
  const JwParams p = collect_params(j, j->last_epoch);
  k_jwin_mark<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t.j, j->t.win, p, eof);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return collect_flush(j, p, j->nq);
}

bw_status bw_collect_advance(bw_collect* j, int64_t system_now_us, bw_collect_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  COLLECT_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > j->now) j->now = system_now_us;
    bw_status st = collect_wake(j, 0);
    if (st != BW_OK) return st;
  }
  return collect_collect(j, out);
}

bw_status bw_collect_eof(bw_collect* j, bw_collect_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  COLLECT_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = collect_wake(j, 1);
  if (st != BW_OK) return st;
  return collect_collect(j, out);
}

// ===========================================================================
// K10 host side: windowed join over session windows (bw_sjwin.cuh)
// ===========================================================================
struct bw_sjwin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_sjwin_spec spec{};
  SjTable t{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;                 // err, why
  unsigned long long* d_cnt = nullptr;  // down, meta, late, released, carried-over queue entries, merged ids
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_side = nullptr, *d_late = nullptr;
  u64* d_handles = nullptr;
  i64* d_ts = nullptr;
  SjEmit e{};
  JwPool pool{}, pool2{};  // ordered mode: the queue, and the one the next flush writes
  u64 nq = 0;              // entries in `pool`
  int slot_bits = 1;
  SortScratch srt;       // pool sort and ordering scratch
  HostCols hd[2];        // down: key, window id, h0, h1, h2 | h3, mask, epoch
  HostCols hm[2];        // meta: key, window id, open, close, epoch | merged count, merged offset
  HostCols hl;           // late: key, window id, epoch, activation, row
  i64* h_mids = nullptr;
  std::vector<u64> merged_off;
  std::vector<i64> merged_ids;
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;     // a call whose released handles and queue count are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
};

bw_status bw_sjwin_create(bw_ctx* ctx, const bw_sjwin_spec* spec, bw_sjwin** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_sjwin_create: NULL argument");
  if (spec->struct_size != sizeof(bw_sjwin_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_sjwin_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "session joins run on one GPU (world == 1)");
  if (spec->insert_mode != BW_JOIN_INSERT_FIRST && spec->insert_mode != BW_JOIN_INSERT_LAST)
    CTX_FAIL(ctx, BW_ERR_SPEC, "insert_mode must be first or last (product: host engine)");
  if (spec->emit_mode < BW_JOIN_EMIT_COMPLETE || spec->emit_mode > BW_JOIN_EMIT_RUNNING) CTX_FAIL(ctx, BW_ERR_SPEC, "bad emit_mode");
  if (spec->ordered != 0 && spec->ordered != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "ordered must be 0 or 1");
  if (spec->sides < 1 || spec->sides > BW_JW_MAXSIDES) CTX_FAIL(ctx, BW_ERR_SPEC, "sides must be in 1..%d", BW_JW_MAXSIDES);
  if (spec->max_sessions_per_key < 1 || spec->max_sessions_per_key > BW_SESS_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_sessions_per_key must be in 1..%d", BW_SESS_MAXM);
  if (spec->gap_us < 0 || spec->gap_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "gap_us must be in 0..UTC_MAX - UTC_MIN");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_queued_rows >= (1ULL << 31) - spec->max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "max_queued_rows + max_batch_rows must stay below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_sjwin, void (*)(bw_sjwin*)> jp(new bw_sjwin(), bw_sjwin_destroy);  // torn down on every failure
  bw_sjwin* j = jp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_sessions_per_key;
  SjTable& t = j->t;
  t.cap = cap;
  t.M = M;
  t.sides = spec->sides;
  t.gap = spec->gap_us;
  while ((1ULL << j->slot_bits) < cap + 1) ++j->slot_bits;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.keys, cap + 1));
  CU(ctx, own.dev(&t.st, cap + 1));
  CU(ctx, own.dev(&t.kx, cap + 1));
  CU(ctx, own.dev(&t.rec, (cap + 1) * (u64)M));
  CU(ctx, own.dev(&t.mrg, (cap + 1) * (u64)(2 * M)));
  t.win = nullptr;  // (K8's window records: sessions live in rec)
  CU(ctx, own.dev(&t.err, 2));
  t.why = t.err + 1;
  CU(ctx, own.dev(&j->d_cnt, 6));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 48, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 64 / sizeof(unsigned long long)));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  const u64 q = spec->ordered ? spec->max_queued_rows : 0;
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_side, n));
  CU(ctx, own.dev(&j->d_late, n));
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_ts, n));
  if (spec->ordered) {
    if ((st = jwin_pool_alloc(ctx, own, j->pool, q + n)) != BW_OK) return st;
    if ((st = jwin_pool_alloc(ctx, own, j->pool2, q + n)) != BW_OK) return st;
  }
  SjEmit& e = j->e;
  for (u64** c : {&e.key, &e.wid, &e.h0, &e.h1, &e.h2, &e.h3, &e.mask, &e.epoch, &e.ord, &e.seq}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.m_key, &e.m_wid, &e.m_epoch, &e.m_ord, &e.m_seq, &e.m_moff, &e.m_mcnt}) CU(ctx, own.dev(c, m));
  for (i64** c : {&e.m_open, &e.m_close, &e.mids}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  // the release buffer grows with the handles held (jwin_room); it starts at one batch
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.max_queue = q;
  e.n_rows = j->d_cnt;
  e.n_meta = j->d_cnt + 1;
  e.n_late = j->d_cnt + 2;
  e.n_rel = j->d_cnt + 3;
  e.n_next = j->d_cnt + 4;
  e.n_mids = j->d_cnt + 5;
  const u64 ns = std::max(std::max(m, l), q + n);
  CU(ctx, j->srt.reserve(own, ns, ns, j->s));
  CU(ctx, j->hd[0].reserve(own, m, m));
  CU(ctx, j->hd[1].reserve(own, m, m));
  CU(ctx, j->hm[0].reserve(own, m, m));
  CU(ctx, j->hm[1].reserve(own, m, m));
  CU(ctx, j->hl.reserve(own, l, l));
  CU(ctx, own.host(&j->h_mids, m));
  k_sjwin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = jp.release();
  return BW_OK;
}

void bw_sjwin_destroy(bw_sjwin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static JwParams sjwin_params(bw_sjwin* j, u64 epoch) {
  JwParams p{};
  p.insert_last = j->spec.insert_mode == BW_JOIN_INSERT_LAST;
  p.emit_mode = j->spec.emit_mode;
  p.ordered = j->spec.ordered;
  p.wait = j->spec.wait_us;
  p.now = j->now;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.batch_no = j->batch_no;
  return p;
}

static const char* jwin_what(const bw_sjwin*) { return "session join"; }
static const char* jwin_full_windows(const bw_sjwin*) { return " a key needs more than max_sessions_per_key sessions or merged ids;"; }
static const char* jwin_full_emit(const bw_sjwin*) { return " more than max_emit_rows down or meta rows or merged ids since the last advance;"; }
static u64 jwin_counters(const bw_sjwin*) { return 6; }  // K8's five, then merged ids

#define SJWIN_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "session join: an earlier call failed on the device; the join is unusable")

// ordered mode: K8's pool sort and flush with the session flush kernel
static bw_status sjwin_flush_pool(bw_sjwin* j, const JwParams& p, u64 n) {
  return jwin_flush_pool(j, p, n, [&](const SjEmit& e, const u32* perm) {
    k_sjwin_flush<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, p, j->pool, perm);
  });
}

bw_status bw_sjwin_apply_device(bw_sjwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles, const int64_t* d_ts_us,
                                uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SJWIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "session join: rows > max_batch_rows");
  if (rows && (!d_keys || !d_side || !d_handles || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "session join: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "session join: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = sjwin_params(j, epoch);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = jwin_room(j, rows)) != BW_OK) return st;
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_sjwin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, d_handles,
                                                     d_side, d_ts_us, j->d_late, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return sjwin_flush_pool(j, p, j->nq + rows);
  return BW_OK;
}

bw_status bw_sjwin_apply(bw_sjwin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us, uint64_t rows,
                         uint64_t epoch, int64_t system_now_us) {
  return jwin_apply_host(j, keys, side, handles, ts_us, rows, epoch, system_now_us, bw_sjwin_apply_device);
}

static bw_status sjwin_collect(bw_sjwin* j, bw_sjwin_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 48, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 nd = j->h_cnt[0], nm = j->h_cnt[1], nl = j->h_cnt[2], nmid = j->h_cnt[5];  // all within bounds: jwin_drain passed
  const SjEmit& e = j->e;
  const u64* down[] = {e.key, e.wid, e.h0, e.h1, e.h2, e.h3, e.mask, e.epoch};
  const u64* meta[] = {e.m_key, e.m_wid, (const u64*)e.m_open, (const u64*)e.m_close, e.m_epoch, e.m_mcnt, e.m_moff};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(j, nd, e.key, e.seq, e.ord, down, 8, j->hd)) != BW_OK) return st;
  if ((st = jwin_ship(j, nm, e.m_key, e.m_seq, e.m_ord, meta, 7, j->hm)) != BW_OK) return st;
  if ((st = jwin_ship(j, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &j->hl)) != BW_OK) return st;
  if (nmid) CU(ctx, cudaMemcpyAsync(j->h_mids, e.mids, nmid * 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 24, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 5, 0, 8, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  // merged ids in meta row order
  j->merged_off.assign(nm + 1, 0);
  j->merged_ids.resize(nmid);
  const u64 *cnt = j->hm[1].col[0], *off = j->hm[1].col[1];
  for (u64 r = 0; r < nm; ++r) {
    j->merged_off[r + 1] = j->merged_off[r] + cnt[r];
    std::copy(j->h_mids + off[r], j->h_mids + off[r] + cnt[r], j->merged_ids.begin() + j->merged_off[r]);
  }
  j->first_call = j->calls;
  out->n_down = nd;
  out->down_key = j->hd[0].col[0];
  out->down_window_id = (const int64_t*)j->hd[0].col[1];
  out->down_handle[0] = j->hd[0].col[2];
  out->down_handle[1] = j->hd[0].col[3];
  out->down_handle[2] = j->hd[0].col[4];
  out->down_handle[3] = j->hd[1].col[0];
  out->down_mask = j->hd[1].col[1];
  out->down_epoch = j->hd[1].col[2];
  out->n_meta = nm;
  out->meta_key = j->hm[0].col[0];
  out->meta_window_id = (const int64_t*)j->hm[0].col[1];
  out->meta_open_us = (const int64_t*)j->hm[0].col[2];
  out->meta_close_us = (const int64_t*)j->hm[0].col[3];
  out->meta_epoch = j->hm[0].col[4];
  out->merged_off = j->merged_off.data();
  out->merged_ids = j->merged_ids.data();
  out->n_late = nl;
  out->late_key = j->hl.col[0];
  out->late_epoch = j->hl.col[2];
  out->late_activation = j->hl.col[3];
  out->late_row = j->hl.col[4];
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys (K8's k_jwin_mark with the session notify_at), then flush them (ordered: through
// the pool)
static bw_status sjwin_wake(bw_sjwin* j, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = jwin_drain(j);
  if (st != BW_OK) return st;
  if ((st = jwin_room(j, 0)) != BW_OK) return st;
  const JwParams p = sjwin_params(j, j->last_epoch);
  k_jwin_mark<<<ctx->sm_count * 8, 256, 0, j->s>>>((const JwTable&)j->t, (const SjRec*)j->t.rec, p, eof, SjNotifyAt{j->t.gap});
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return sjwin_flush_pool(j, p, j->nq);
  k_sjwin_flush<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, p, j->pool, nullptr);
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

bw_status bw_sjwin_advance(bw_sjwin* j, int64_t system_now_us, bw_sjwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SJWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > j->now) j->now = system_now_us;
    bw_status st = sjwin_wake(j, 0);
    if (st != BW_OK) return st;
  }
  return sjwin_collect(j, out);
}

bw_status bw_sjwin_eof(bw_sjwin* j, bw_sjwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SJWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = sjwin_wake(j, 1);
  if (st != BW_OK) return st;
  return sjwin_collect(j, out);
}

// ===========================================================================
// K12 host side: collect_window over session windows (bw_scwin.cuh)
// ===========================================================================
// K9's store, staging, output and growth (collect_room, collect_place) and K8's drain and release-buffer growth
// (jwin_drain, jwin_room) read these members by the names bw_collect / bw_jwin give them.
struct bw_scwin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_scwin_spec spec{};
  ScTable t{};
  CwStore es{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;  // err, why
  // closed sessions, merged ids, late rows, released, carried-over queue entries, staged, store, intervals, merges
  unsigned long long* d_cnt = nullptr;
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_late = nullptr, *d_flag = nullptr;
  u64* d_handles = nullptr;
  i64* d_ts = nullptr;
  ScEmit e{};
  JwPool pool{}, pool2{};  // ordered mode: the queue, and the one the next flush writes
  u64 nq = 0;              // entries in `pool`
  int slot_bits = 1;
  u64 kmax = 1;            // entries one value adds: it joins one session
  u64 n_store = 0, dead = 0;    // entries in the store, and how many of them are dead
  u64 n_rows = 0, n_stage = 0;  // closed sessions and staged handles since the last advance / eof
  u64 n_mrg = 0;                // merges applied so far
  SortScratch srt;              // pool sort, ordering and compaction scratch
  u32* d_inv = nullptr;         // advance / eof: a closed session's place in the reference's order
  u64 *d_cs = nullptr, *d_off = nullptr;  // its count in that order, and the exclusive scan of them
  u64* d_out = nullptr;         // the handles in the reference's order
  u64* h_out = nullptr;
  u64 out_cap = 0;
  HostCols hd[2];  // down: key, id, epoch, open, close | merged count, merged offset, interval count, interval offset, CSR
  HostCols hl;     // late: key, window id, epoch, activation, row
  i64* h_mids = nullptr;
  u64* h_ivs = nullptr;
  std::vector<u64> merged_off, merge_off, merge_start, merge_end;
  std::vector<i64> merged_ids;
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;     // a call whose counts are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
};

bw_status bw_scwin_create(bw_ctx* ctx, const bw_scwin_spec* spec, bw_scwin** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_scwin_create: NULL argument");
  if (spec->struct_size != sizeof(bw_scwin_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_scwin_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "session collects run on one GPU (world == 1)");
  if (spec->ordered != 0 && spec->ordered != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "ordered must be 0 or 1");
  if (spec->max_sessions_per_key < 1 || spec->max_sessions_per_key > BW_SESS_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_sessions_per_key must be in 1..%d", BW_SESS_MAXM);
  if (spec->gap_us < 0 || spec->gap_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "gap_us must be in 0..UTC_MAX - UTC_MIN");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_queued_rows >= (1ULL << 31) - spec->max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "max_queued_rows + max_batch_rows must stay below 2^31");
  if (spec->max_emit_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "max_emit_rows must be below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_scwin, void (*)(bw_scwin*)> cp(new bw_scwin(), bw_scwin_destroy);  // torn down on every failure
  bw_scwin* j = cp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_sessions_per_key;
  const u64 cells = (cap + 1) * (u64)M;
  ScTable& t = j->t;
  t.j.cap = cap;
  t.j.M = M;
  t.j.sides = 1;
  t.gap = spec->gap_us;
  while ((1ULL << j->slot_bits) < cap + 1) ++j->slot_bits;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.j.keys, cap + 1));
  CU(ctx, own.dev(&t.j.st, cap + 1));
  CU(ctx, own.dev(&t.kx, cap + 1));
  CU(ctx, own.dev(&t.rec, cells));
  CU(ctx, own.dev(&t.mrg, 2 * cells));
  CU(ctx, own.dev(&t.iv, cells));
  CU(ctx, own.dev(&t.cell_ord, cells));
  CU(ctx, own.dev(&t.cell_c, cells));
  CU(ctx, own.dev(&t.cell_mord, cells));
  CU(ctx, own.dev(&t.cell_root, cells));
  CU(ctx, own.dev(&t.cell_base, cells));
  t.j.win = nullptr;  // (K8's window records: sessions live in rec)
  t.win = nullptr;
  CU(ctx, own.dev(&t.j.err, 2));
  t.j.why = t.j.err + 1;
  t.err = t.j.err;
  t.why = t.j.why;
  CU(ctx, own.dev(&j->d_cnt, 9));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 72, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 128 / sizeof(unsigned long long)));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  const u64 q = spec->ordered ? spec->max_queued_rows : 0;
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_late, n));
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_ts, n));
  if (spec->ordered) {
    if ((st = jwin_pool_alloc(ctx, own, j->pool, q + n)) != BW_OK) return st;
    if ((st = jwin_pool_alloc(ctx, own, j->pool2, q + n)) != BW_OK) return st;
  }
  ScEmit& e = j->e;
  for (u64** c : {&e.key, &e.wid, &e.cnt, &e.soff, &e.epoch, &e.ord, &e.seq, &e.moff, &e.mcnt, &e.ioff, &e.icnt, &e.ivs}) CU(ctx, own.dev(c, m));
  for (i64** c : {&e.open, &e.close, &e.mids}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  CU(ctx, own.dev(&j->d_inv, m));
  CU(ctx, own.dev(&j->d_cs, m + 1));
  CU(ctx, own.dev(&j->d_off, m + 1));
  // the store, the staging buffer, the output and the release buffer grow with what the collect holds (collect_room);
  // they start at one batch
  CwStore& es = j->es;
  es.cap = n;
  CU(ctx, own.dev(&es.ref, n));
  CU(ctx, own.dev(&es.rank, n));
  CU(ctx, own.dev(&es.h, n));
  CU(ctx, own.dev(&j->d_flag, n));
  e.max_stage = n;
  CU(ctx, own.dev(&e.stage, n));
  CU(ctx, own.dev(&e.stage_rec, n));
  j->out_cap = n;
  CU(ctx, own.dev(&j->d_out, n));
  CU(ctx, own.host(&j->h_out, n));
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.max_queue = q;
  e.n_rows = j->d_cnt;
  e.n_mids = j->d_cnt + 1;
  e.n_late = j->d_cnt + 2;
  e.n_rel = j->d_cnt + 3;   // (jwin_drain reads these two)
  e.n_next = j->d_cnt + 4;
  e.n_stage = j->d_cnt + 5;
  es.n = j->d_cnt + 6;
  e.n_ivs = j->d_cnt + 7;
  e.n_mrg = j->d_cnt + 8;
  const u64 ns = std::max(std::max(m, l), q + n);
  CU(ctx, j->srt.reserve(own, ns, ns, j->s));
  size_t b = 0;
  CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b, j->d_cs, j->d_off, (int)(m + 1), j->s));
  CU(ctx, j->srt.grow_cub(own, b + 256));
  CU(ctx, j->hd[0].reserve(own, m, m));
  CU(ctx, j->hd[1].reserve(own, m + 1, m + 1));
  CU(ctx, j->hl.reserve(own, l, l));
  CU(ctx, own.host(&j->h_mids, m));
  CU(ctx, own.host(&j->h_ivs, m));
  k_scwin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = cp.release();
  return BW_OK;
}

void bw_scwin_destroy(bw_scwin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static JwParams scwin_params(bw_scwin* j, u64 epoch) {
  JwParams p{};
  p.ordered = j->spec.ordered;
  p.wait = j->spec.wait_us;
  p.now = j->now;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.batch_no = j->batch_no;
  return p;
}

static const char* jwin_what(const bw_scwin*) { return "session collect"; }
static const char* jwin_full_windows(const bw_scwin*) {
  return " a key needs more than max_sessions_per_key sessions, merged ids or merge intervals;";
}
static const char* jwin_full_emit(const bw_scwin*) {
  return " more than max_emit_rows closed sessions, merged ids or merge intervals since the last advance;";
}
static u64 jwin_counters(const bw_scwin*) { return 9; }

#define SCWIN_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "session collect: an earlier call failed on the device; the collect is unusable")

// K8's drain (fail on a device-side overflow, take the released handles and the queue count), then the store's counts
static bw_status scwin_drain(bw_scwin* j) {
  const bool fresh = j->undrained;
  bw_status st = jwin_drain(j);
  if (st != BW_OK || !fresh) return st;
  j->n_rows = j->h_cnt[0];
  j->dead += j->h_cnt[5] - j->n_stage;  // every staged handle left a dead entry behind
  j->n_stage = j->h_cnt[5];
  j->n_store = j->h_cnt[6];
  j->n_mrg = j->h_cnt[8];
  return BW_OK;
}

// after the per-key kernels of a call: retag the merged-away sessions' entries, move the closed sessions' out
static bw_status scwin_gather(bw_scwin* j, const JwParams& p) {
  k_scwin_gather<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->n_rows, j->n_mrg);
  CU(j->ctx, cudaGetLastError());
  return BW_OK;
}

// K8's pool sort (ordered), then every woken key's flush (k_scwin_flush), then the gather
static bw_status scwin_flush(bw_scwin* j, const JwParams& p, u64 n) {
  bw_ctx* ctx = j->ctx;
  bw_status st = j->spec.ordered ? jwin_sort_pool(j, j->t.j, p, n) : BW_OK;
  if (st != BW_OK) return st;
  ScEmit e = j->e;
  e.next = j->pool2;
  k_scwin_flush<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, j->es, p, j->pool, j->srt.perm);
  CU(ctx, cudaGetLastError());
  if (j->spec.ordered) std::swap(j->pool, j->pool2);  // the next call reads what this flush carried over (count: the drain)
  return scwin_gather(j, p);
}

bw_status bw_scwin_apply_device(bw_scwin* j, const uint64_t* d_keys, const uint64_t* d_handles, const int64_t* d_ts_us, uint64_t rows,
                                uint64_t epoch, int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SCWIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "session collect: rows > max_batch_rows");
  if (rows && (!d_keys || !d_handles || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "session collect: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "session collect: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = scwin_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = scwin_params(j, epoch);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = collect_room(j, rows)) != BW_OK) return st;
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_scwin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted, j->k.d_head,
                                                     d_handles, d_ts_us, j->d_late, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return scwin_flush(j, p, j->nq + rows);
  return scwin_gather(j, p);
}

bw_status bw_scwin_apply(bw_scwin* j, const uint64_t* keys, const uint64_t* handles, const int64_t* ts_us, uint64_t rows, uint64_t epoch,
                         int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "session collect: rows > max_batch_rows");
  if (rows && (!keys || !handles || !ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "session collect: NULL column");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = scwin_drain(j);
  if (st != BW_OK) return st;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, j->s));
  }
  st = bw_scwin_apply_device(j, j->k.d_keys, j->d_handles, j->d_ts, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return scwin_drain(j);
}

static bw_status scwin_collect(bw_scwin* j, bw_scwin_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = scwin_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 72, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  // all within bounds: the drain passed
  const u64 nd = j->h_cnt[0], nmid = j->h_cnt[1], nl = j->h_cnt[2], ns = j->h_cnt[5], niv = j->h_cnt[7];
  const ScEmit& e = j->e;
  const u64* down[] = {e.key, e.wid, e.epoch, (const u64*)e.open, (const u64*)e.close, e.mcnt, e.moff, e.icnt, e.ioff};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(j, nd, e.key, e.seq, e.ord, down, 9, j->hd)) != BW_OK) return st;
  if ((st = collect_place(j, nd, ns, j->hd[1].col[4])) != BW_OK) return st;
  if ((st = jwin_ship(j, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &j->hl)) != BW_OK) return st;
  if (nmid) CU(ctx, cudaMemcpyAsync(j->h_mids, e.mids, nmid * 8, cudaMemcpyDeviceToHost, j->s));
  if (niv) CU(ctx, cudaMemcpyAsync(j->h_ivs, e.ivs, niv * 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 24, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 5, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 7, 0, 8, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  // merged ids and intervals in down row order
  j->merged_off.assign(nd + 1, 0);
  j->merged_ids.resize(nmid);
  j->merge_off.assign(nd + 1, 0);
  j->merge_start.resize(niv);
  j->merge_end.resize(niv);
  const u64 *mcnt = j->hd[1].col[0], *moff = j->hd[1].col[1], *icnt = j->hd[1].col[2], *ioff = j->hd[1].col[3];
  for (u64 r = 0; r < nd; ++r) {
    j->merged_off[r + 1] = j->merged_off[r] + mcnt[r];
    std::copy(j->h_mids + moff[r], j->h_mids + moff[r] + mcnt[r], j->merged_ids.begin() + j->merged_off[r]);
    j->merge_off[r + 1] = j->merge_off[r] + icnt[r];
    for (u64 k = 0; k < icnt[r]; ++k) {
      const u64 v = j->h_ivs[ioff[r] + k];
      j->merge_start[j->merge_off[r] + k] = v >> 32;
      j->merge_end[j->merge_off[r] + k] = v & 0xffffffffULL;
    }
  }
  j->n_rows = j->n_stage = 0;
  j->first_call = j->calls;
  out->n_down = nd;
  out->down_key = j->hd[0].col[0];
  out->down_window_id = (const int64_t*)j->hd[0].col[1];
  out->down_epoch = j->hd[0].col[2];
  out->down_offset = j->hd[1].col[4];
  out->handle = j->h_out;
  out->open_us = (const int64_t*)j->hd[0].col[3];
  out->close_us = (const int64_t*)j->hd[0].col[4];
  out->merged_off = j->merged_off.data();
  out->merged_ids = j->merged_ids.data();
  out->merge_off = j->merge_off.data();
  out->merge_start = j->merge_start.data();
  out->merge_end = j->merge_end.data();
  out->n_late = nl;
  out->late_key = j->hl.col[0];
  out->late_epoch = j->hl.col[2];
  out->late_activation = j->hl.col[3];
  out->late_row = j->hl.col[4];
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys (K8's k_jwin_mark with the session notify_at), then flush them (ordered: through
// the pool)
static bw_status scwin_wake(bw_scwin* j, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = scwin_drain(j);
  if (st != BW_OK) return st;
  if ((st = collect_room(j, 0)) != BW_OK) return st;
  const JwParams p = scwin_params(j, j->last_epoch);
  k_jwin_mark<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t.j, (const ScRec*)j->t.rec, p, eof, SjNotifyAt{j->t.gap});
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return scwin_flush(j, p, j->nq);
}

bw_status bw_scwin_advance(bw_scwin* j, int64_t system_now_us, bw_scwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SCWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > j->now) j->now = system_now_us;
    bw_status st = scwin_wake(j, 0);
    if (st != BW_OK) return st;
  }
  return scwin_collect(j, out);
}

bw_status bw_scwin_eof(bw_scwin* j, bw_scwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SCWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = scwin_wake(j, 1);
  if (st != BW_OK) return st;
  return scwin_collect(j, out);
}

// ===========================================================================
// K11 host side: windowed arg-max / arg-min (bw_argwin.cuh)
// ===========================================================================
struct bw_argwin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_argwin_spec spec{};
  AwTable t{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;                 // err, why
  unsigned long long* d_cnt = nullptr;  // closed rows, merged ids, late, released, (unused: K8's queue count)
  unsigned long long* h_cnt = nullptr;
  u64 *d_handles = nullptr, *d_by = nullptr;
  i64* d_ts = nullptr;
  AwEmit e{};
  u64 nq = 0;            // (no queue: jwin_drain's count, always 0)
  SortScratch srt;       // ordering scratch
  HostCols hd[2];        // closed: key, window id, handle, open, close | epoch, merged count, merged offset
  HostCols hl;           // late: key, window id, epoch, activation, row
  i64* h_mids = nullptr;
  std::vector<u64> merged_off;
  std::vector<i64> merged_ids;
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;     // a call whose released handles are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
};

// what the host steps K11 shares with the handle joins (jwin_drain, jwin_room, jwin_ship) ask of it
static const char* jwin_what(const bw_argwin*) { return "windowed arg-max / arg-min"; }
static const char* jwin_full_windows(const bw_argwin* a) {
  return a->spec.session ? " a key needs more than max_windows_per_key sessions or merged ids;" : " a key needs more than max_windows_per_key open windows;";
}
static const char* jwin_full_emit(const bw_argwin*) { return " more than max_emit_rows closed rows or merged ids since the last advance;"; }
static u64 jwin_counters(const bw_argwin*) { return 5; }
static bool jwin_queues(const bw_argwin*) { return false; }

bw_status bw_argwin_create(bw_ctx* ctx, const bw_argwin_spec* spec, bw_argwin** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_argwin_create: NULL argument");
  if (spec->struct_size != sizeof(bw_argwin_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_argwin_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed arg-max / arg-min run on one GPU (world == 1)");
  if (spec->extreme != BW_RED_MAX && spec->extreme != BW_RED_MIN) CTX_FAIL(ctx, BW_ERR_SPEC, "extreme must be BW_RED_MAX or BW_RED_MIN");
  if (spec->by_dtype != BW_VAL_I64 && spec->by_dtype != BW_VAL_F64) CTX_FAIL(ctx, BW_ERR_SPEC, "by_dtype must be BW_VAL_I64 or BW_VAL_F64");
  if (spec->session != 0 && spec->session != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "session must be 0 or 1");
  if (spec->max_windows_per_key < 1 || spec->max_windows_per_key > BW_JW_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_windows_per_key must be in 1..%d", BW_JW_MAXM);
  if (spec->session) {
    if (spec->gap_us < 0 || spec->gap_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "gap_us must be in 0..UTC_MAX - UTC_MIN");
  } else {
    if (spec->length_us <= 0 || spec->length_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "length_us must be in 1..UTC_MAX - UTC_MIN");
    if (spec->offset_us <= 0 || spec->offset_us > spec->length_us) CTX_FAIL(ctx, BW_ERR_SPEC, "offset_us must be in 1..length_us");
    if (spec->align_us < BW_UTC_MIN_US || spec->align_us > BW_UTC_MAX_US) CTX_FAIL(ctx, BW_ERR_SPEC, "align_us out of range");
  }
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_argwin, void (*)(bw_argwin*)> ap(new bw_argwin(), bw_argwin_destroy);  // torn down on every failure
  bw_argwin* a = ap.get();
  Owner& own = a->own;
  a->ctx = ctx;
  a->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_windows_per_key;
  AwTable& t = a->t;
  t.j.cap = cap;
  t.j.M = M;
  t.j.sides = 1;
  t.gap = spec->gap_us;
  t.is_max = spec->extreme == BW_RED_MAX;
  t.is_f64 = spec->by_dtype == BW_VAL_F64;
  CU(ctx, own.stream(&a->s));
  CU(ctx, own.dev(&t.j.keys, cap + 1));
  CU(ctx, own.dev(&t.j.st, cap + 1));
  if (spec->session) {
    CU(ctx, own.dev(&t.kx, cap + 1));
    CU(ctx, own.dev(&t.rec, (cap + 1) * (u64)M));
    CU(ctx, own.dev(&t.mrg, (cap + 1) * (u64)(2 * M)));
  } else {
    CU(ctx, own.dev(&t.win, (cap + 1) * (u64)M));
  }
  CU(ctx, own.dev(&t.j.err, 2));
  t.j.why = t.j.err + 1;
  t.err = t.j.err;
  t.why = t.j.why;
  CU(ctx, own.dev(&a->d_cnt, 5));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, a->s));
  CU(ctx, cudaMemsetAsync(a->d_cnt, 0, 40, a->s));
  CU(ctx, own.host(&a->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&a->h_cnt, 64 / sizeof(unsigned long long)));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  bw_status st = keyed_alloc(ctx, own, a->k, n, a->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&a->d_handles, n));
  CU(ctx, own.dev(&a->d_by, n));
  CU(ctx, own.dev(&a->d_ts, n));
  AwEmit& e = a->e;
  for (u64** c : {&e.key, &e.wid, &e.h, &e.epoch, &e.ord, &e.seq, &e.moff, &e.mcnt}) CU(ctx, own.dev(c, m));
  for (i64** c : {&e.open, &e.close, &e.mids}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  // the release buffer grows with the handles held (jwin_room); it starts at one batch
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.n_rows = a->d_cnt;
  e.n_mids = a->d_cnt + 1;
  e.n_late = a->d_cnt + 2;
  e.n_rel = a->d_cnt + 3;
  const u64 ns = std::max(m, l);
  CU(ctx, a->srt.reserve(own, ns, ns, a->s));
  CU(ctx, a->hd[0].reserve(own, m, m));
  CU(ctx, a->hd[1].reserve(own, m, m));
  CU(ctx, a->hl.reserve(own, l, l));
  CU(ctx, own.host(&a->h_mids, m));
  k_awin_init<<<ctx->sm_count * 4, 256, 0, a->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(a->s));
  *out = ap.release();
  return BW_OK;
}

void bw_argwin_destroy(bw_argwin* a) {
  if (!a) return;
  cudaSetDevice(a->ctx->device);
  if (a->s) cudaStreamSynchronize(a->s);
  delete a;  // a->own releases every buffer and the stream
}

static JwParams argwin_params(bw_argwin* a, u64 epoch) {
  JwParams p{};
  p.length = a->spec.length_us;
  p.offset = a->spec.offset_us;
  p.align = a->spec.align_us;
  p.wait = a->spec.wait_us;
  p.now = a->now;
  p.epoch = epoch;
  p.ord = a->calls++;
  p.batch_no = a->batch_no;
  return p;
}

bw_status bw_argwin_apply_device(bw_argwin* a, const uint64_t* d_keys, const uint64_t* d_handles, const uint64_t* d_by_bits,
                                 const int64_t* d_ts_us, uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (!a) return BW_ERR_SPEC;
  bw_ctx* ctx = a->ctx;
  if (rows > a->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed arg-max / arg-min: rows > max_batch_rows");
  if (rows && (!d_keys || !d_handles || !d_by_bits || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed arg-max / arg-min: NULL column");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = jwin_drain(a);
  if (st != BW_OK) return st;
  if (a->batch_no && epoch < a->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "windowed arg-max / arg-min: epochs must not decrease");
  a->last_epoch = epoch;
  if (system_now_us > a->now) a->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = argwin_params(a, epoch);
  a->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = jwin_room(a, rows)) != BW_OK) return st;
  a->outstanding += rows;
  st = keyed_group(ctx, a->k, d_keys, rows, a->s);
  if (st != BW_OK) return st;
  if (a->spec.session)
    k_aswin_apply<<<ctx->sm_count * 8, 256, 0, a->s>>>(a->t, a->e, p, a->k.d_ksorted, a->k.d_isorted, a->k.d_head, d_handles, d_by_bits,
                                                       d_ts_us, rows);
  else
    k_awin_apply<<<ctx->sm_count * 8, 256, 0, a->s>>>(a->t, a->e, p, a->k.d_ksorted, a->k.d_isorted, a->k.d_head, d_handles, d_by_bits,
                                                      d_ts_us, rows);
  CU(ctx, cudaGetLastError());
  a->undrained = true;
  return BW_OK;
}

bw_status bw_argwin_apply(bw_argwin* a, const uint64_t* keys, const uint64_t* handles, const uint64_t* by_bits, const int64_t* ts_us,
                          uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (!a) return BW_ERR_SPEC;
  bw_ctx* ctx = a->ctx;
  if (rows > a->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed arg-max / arg-min: rows > max_batch_rows");
  if (rows && (!keys || !handles || !by_bits || !ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed arg-max / arg-min: NULL column");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = jwin_drain(a);
  if (st != BW_OK) return st;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(a->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, a->s));
    CU(ctx, cudaMemcpyAsync(a->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, a->s));
    CU(ctx, cudaMemcpyAsync(a->d_by, by_bits, rows * 8, cudaMemcpyHostToDevice, a->s));
    CU(ctx, cudaMemcpyAsync(a->d_ts, ts_us, rows * 8, cudaMemcpyHostToDevice, a->s));
  }
  st = bw_argwin_apply_device(a, a->k.d_keys, a->d_handles, a->d_by, a->d_ts, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return jwin_drain(a);
}

static bw_status argwin_collect(bw_argwin* a, bw_argwin_rows* out) {
  bw_ctx* ctx = a->ctx;
  bw_status st = jwin_drain(a);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(a->h_cnt, a->d_cnt, 24, cudaMemcpyDeviceToHost, a->s));
  CU(ctx, cudaStreamSynchronize(a->s));
  const u64 nc = a->h_cnt[0], nmid = a->h_cnt[1], nl = a->h_cnt[2];  // all within bounds: jwin_drain passed
  const AwEmit& e = a->e;
  const u64* closed[] = {e.key, e.wid, e.h, (const u64*)e.open, (const u64*)e.close, e.epoch, e.mcnt, e.moff};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(a, nc, e.key, e.seq, e.ord, closed, 8, a->hd)) != BW_OK) return st;
  if ((st = jwin_ship(a, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &a->hl)) != BW_OK) return st;
  if (nmid) CU(ctx, cudaMemcpyAsync(a->h_mids, e.mids, nmid * 8, cudaMemcpyDeviceToHost, a->s));
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(a->d_cnt, 0, 24, a->s));
  CU(ctx, cudaStreamSynchronize(a->s));
  // merged ids in closed row order
  a->merged_off.assign(nc + 1, 0);
  a->merged_ids.resize(nmid);
  const u64 *cnt = a->hd[1].col[1], *off = a->hd[1].col[2];
  for (u64 r = 0; r < nc; ++r) {
    a->merged_off[r + 1] = a->merged_off[r] + cnt[r];
    std::copy(a->h_mids + off[r], a->h_mids + off[r] + cnt[r], a->merged_ids.begin() + a->merged_off[r]);
  }
  a->first_call = a->calls;
  out->n_closed = nc;
  out->closed_key = a->hd[0].col[0];
  out->closed_window_id = (const int64_t*)a->hd[0].col[1];
  out->closed_handle = a->hd[0].col[2];
  out->closed_open_us = (const int64_t*)a->hd[0].col[3];
  out->closed_close_us = (const int64_t*)a->hd[0].col[4];
  out->closed_epoch = a->hd[1].col[0];
  out->merged_off = a->merged_off.data();
  out->merged_ids = a->merged_ids.data();
  out->n_late = nl;
  out->late_key = a->hl.col[0];
  out->late_window_id = (const int64_t*)a->hl.col[1];
  out->late_epoch = a->hl.col[2];
  out->late_activation = a->hl.col[3];
  out->late_row = a->hl.col[4];
  // handed out until the next advance / eof, then cleared
  a->released.swap(a->released_out);
  a->released.clear();
  out->n_released = a->released_out.size();
  out->released = a->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys (K8's k_jwin_mark with the windower's notify_at), then close them
static bw_status argwin_wake(bw_argwin* a, int eof) {
  bw_ctx* ctx = a->ctx;
  bw_status st = jwin_drain(a);
  if (st != BW_OK) return st;
  if ((st = jwin_room(a, 0)) != BW_OK) return st;
  const JwParams p = argwin_params(a, a->last_epoch);
  if (a->spec.session)
    k_jwin_mark<<<ctx->sm_count * 8, 256, 0, a->s>>>(a->t.j, (const AwSess*)a->t.rec, p, eof, AwNotifyAt{a->t.gap});
  else
    k_jwin_mark<<<ctx->sm_count * 8, 256, 0, a->s>>>(a->t.j, (const AwWin*)a->t.win, p, eof);
  CU(ctx, cudaGetLastError());
  a->undrained = true;
  k_awin_close<<<ctx->sm_count * 8, 256, 0, a->s>>>(a->t, a->e, p, a->spec.session);
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

bw_status bw_argwin_advance(bw_argwin* a, int64_t system_now_us, bw_argwin_rows* out) {
  if (!a || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = a->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > a->now) a->now = system_now_us;
    bw_status st = argwin_wake(a, 0);
    if (st != BW_OK) return st;
  }
  return argwin_collect(a, out);
}

bw_status bw_argwin_eof(bw_argwin* a, bw_argwin_rows* out) {
  if (!a || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = a->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = argwin_wake(a, 1);
  if (st != BW_OK) return st;
  return argwin_collect(a, out);
}

// ===========================================================================
// K13 host side: keyed collect (bw_kcollect.cuh)
// ===========================================================================
struct bw_kcollect {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_kcollect_spec spec{};
  KcTable t{};
  CwStore es{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;                 // err, why
  unsigned long long* d_cnt = nullptr;  // lists, staged handles, store entries, carried entries moved out
  unsigned long long* h_cnt = nullptr;
  unsigned char* d_flag = nullptr;
  u64* d_handles = nullptr;
  KcSeg* d_seg = nullptr;
  KcEmit e{};
  u64 n_store = 0, dead = 0;      // entries in the store, and how many of them are dead
  u64 n_rows = 0, n_stage = 0;    // lists and staged handles since the last advance / eof
  SortScratch srt;                // ordering and compaction scratch
  u32* d_inv = nullptr;           // advance / eof: a list's place in the reference's order
  u64 *d_cs = nullptr, *d_off = nullptr;  // its count in that order, and the exclusive scan of them
  u64* d_out = nullptr;           // the handles in the reference's order
  u64* h_out = nullptr;
  u64 out_cap = 0;
  HostCols hd;                    // key, epoch, offsets
  bool undrained = false;         // a call whose counts are not read back yet
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  bool failed = false;
};

bw_status bw_kcollect_create(bw_ctx* ctx, const bw_kcollect_spec* spec, bw_kcollect** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_kcollect_create: NULL argument");
  if (spec->struct_size != sizeof(bw_kcollect_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_kcollect_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed collects run on one GPU (world == 1)");
  if (spec->max_size < 1) CTX_FAIL(ctx, BW_ERR_SPEC, "max_size must be at least 1");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_emit_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "max_emit_rows must be below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_kcollect, void (*)(bw_kcollect*)> cp(new bw_kcollect(), bw_kcollect_destroy);  // torn down on every failure
  bw_kcollect* j = cp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  KcTable& t = j->t;
  t.cap = cap;
  t.M = spec->max_size;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.keys, cap + 1));
  CU(ctx, own.dev(&t.cnt, cap + 1));
  CU(ctx, own.dev(&t.due, cap + 1));
  CU(ctx, own.dev(&t.mv_ord, cap + 1));
  CU(ctx, own.dev(&t.mv_base, cap + 1));
  CU(ctx, own.dev(&t.mv_rec, cap + 1));
  CU(ctx, own.dev(&t.err, 2));
  t.why = t.err + 1;
  CU(ctx, own.dev(&j->d_cnt, 4));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 32, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 64 / sizeof(unsigned long long)));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1);
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_seg, n));
  KcEmit& e = j->e;
  for (u64** c : {&e.key, &e.cnt, &e.soff, &e.epoch, &e.ord, &e.seq}) CU(ctx, own.dev(c, m));
  CU(ctx, own.dev(&j->d_inv, m));
  CU(ctx, own.dev(&j->d_cs, m + 1));
  CU(ctx, own.dev(&j->d_off, m + 1));
  // the store, the staging buffer and the output grow with what the collect holds (store_room, collect_place); they
  // start at one batch
  CwStore& es = j->es;
  es.cap = n;
  CU(ctx, own.dev(&es.ref, n));
  CU(ctx, own.dev(&es.rank, n));
  CU(ctx, own.dev(&es.h, n));
  CU(ctx, own.dev(&j->d_flag, n));
  e.max_stage = n;
  CU(ctx, own.dev(&e.stage, n));
  CU(ctx, own.dev(&e.stage_rec, n));
  j->out_cap = n;
  CU(ctx, own.dev(&j->d_out, n));
  CU(ctx, own.host(&j->h_out, n));
  e.max_rows = spec->max_emit_rows;
  e.n_rows = j->d_cnt;
  e.n_stage = j->d_cnt + 1;
  es.n = j->d_cnt + 2;
  e.n_moved = j->d_cnt + 3;
  CU(ctx, j->srt.reserve(own, m, m, j->s));
  size_t b = 0;
  CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b, j->d_cs, j->d_off, (int)(m + 1), j->s));
  CU(ctx, j->srt.grow_cub(own, b + 256));
  CU(ctx, j->hd.reserve(own, m + 1, m + 1));
  k_kcol_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = cp.release();
  return BW_OK;
}

void bw_kcollect_destroy(bw_kcollect* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static KcParams kcollect_params(bw_kcollect* j, u64 epoch, i64 timeout_at) {
  KcParams p;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.timeout_at = timeout_at;
  return p;
}

#define KCOLLECT_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "keyed collect: an earlier call failed on the device; the collect is unusable")

// wait for the last call; fail on a device-side overflow; then take its counts
static bw_status kcollect_drain(bw_kcollect* j) {
  bw_ctx* ctx = j->ctx;
  KCOLLECT_REFUSE_FAILED(j);
  if (!j->undrained) return BW_OK;
  CU(ctx, cudaMemcpyAsync(j->h_err, j->t.err, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 32, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  if (j->h_err[0]) {
    j->failed = true;
    const u32 w = j->h_err[1];
    CTX_FAIL(ctx, (bw_status)j->h_err[0], "keyed collect kernel ran out of capacity:%s%s%s%s",
             w & BW_JW_FULL_TABLE ? " key table full (raise capacity_hint);" : "",
             w & BW_JW_FULL_EMIT ? " more than max_emit_rows lists since the last advance;" : "",
             w & BW_CW_FULL_STORE ? " carry store or staging buffer full;" : "", w ? "" : " (no reason recorded)");
  }
  j->n_rows = j->h_cnt[0];
  j->n_stage = j->h_cnt[1];
  j->n_store = j->h_cnt[2];
  j->dead += j->h_cnt[3];
  CU(ctx, cudaMemsetAsync(j->d_cnt + 3, 0, 8, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->undrained = false;
  return BW_OK;
}

// the carried entries of every key whose carry moved to a list in this call, to their staging slots (k_kcol_gather);
// the store's entries added by this call lie past n_store and are not looked at
static bw_status kcollect_gather(bw_kcollect* j, const KcParams& p) {
  if (j->n_store) k_kcol_gather<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->n_store);
  CU(j->ctx, cudaGetLastError());
  return BW_OK;
}

bw_status bw_kcollect_apply_device(bw_kcollect* j, const uint64_t* d_keys, const uint64_t* d_handles, uint64_t rows, uint64_t epoch,
                                   int64_t timeout_at_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  KCOLLECT_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed collect: rows > max_batch_rows");
  if (rows && (!d_keys || !d_handles)) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed collect: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "keyed collect: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = kcollect_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  const KcParams p = kcollect_params(j, epoch, timeout_at_us);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = store_room(j, rows)) != BW_OK) return st;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  const int grid = ctx->sm_count * 8;
  k_kcol_keys<<<grid, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->d_seg, j->k.d_ksorted, j->k.d_head, rows);
  k_kcol_rows<<<grid, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->d_seg, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, d_handles, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return kcollect_gather(j, p);
}

bw_status bw_kcollect_apply(bw_kcollect* j, const uint64_t* keys, const uint64_t* handles, uint64_t rows, uint64_t epoch,
                            int64_t timeout_at_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed collect: rows > max_batch_rows");
  if (rows && (!keys || !handles)) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed collect: NULL column");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = kcollect_drain(j);
  if (st != BW_OK) return st;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, j->s));
  }
  st = bw_kcollect_apply_device(j, j->k.d_keys, j->d_handles, rows, epoch, timeout_at_us);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return kcollect_drain(j);
}

static bw_status kcollect_collect(bw_kcollect* j, bw_kcollect_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = kcollect_drain(j);
  if (st != BW_OK) return st;
  const u64 nd = j->n_rows, ns = j->n_stage;  // within bounds: kcollect_drain passed
  const KcEmit& e = j->e;
  const u64* cols[] = {e.key, e.epoch};
  if ((st = jwin_ship(j, nd, e.key, e.seq, e.ord, cols, 2, &j->hd)) != BW_OK) return st;
  if ((st = collect_place(j, nd, ns, j->hd.col[2])) != BW_OK) return st;
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 16, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->n_rows = j->n_stage = 0;
  j->first_call = j->calls;
  out->n = nd;
  out->key = j->hd.col[0];
  out->epoch = j->hd.col[1];
  out->offset = j->hd.col[2];
  out->handle = j->h_out;
  return BW_OK;
}

// notify phase or EOF: every due (EOF: every live) key's carry becomes a list
static bw_status kcollect_wake(bw_kcollect* j, i64 now, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = kcollect_drain(j);
  if (st != BW_OK) return st;
  if ((st = store_room(j, 0)) != BW_OK) return st;
  const KcParams p = kcollect_params(j, j->last_epoch, 0);
  k_kcol_due<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, p, now, eof);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return kcollect_gather(j, p);
}

bw_status bw_kcollect_advance(bw_kcollect* j, int64_t now_us, bw_kcollect_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  KCOLLECT_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (now_us > 0) {
    bw_status st = kcollect_wake(j, now_us, 0);
    if (st != BW_OK) return st;
  }
  return kcollect_collect(j, out);
}

bw_status bw_kcollect_eof(bw_kcollect* j, bw_kcollect_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  KCOLLECT_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = kcollect_wake(j, 0, 1);
  if (st != BW_OK) return st;
  return kcollect_collect(j, out);
}

// ===========================================================================
// K14 host side: windowed product join (bw_pjwin.cuh)
// ===========================================================================
struct bw_pjwin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_pjwin_spec spec{};
  PjTable t{};
  PjStore es{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;  // err, why
  // events, meta, late, released, carried-over queue entries, stage records, staged, store entries, values, dead entries
  unsigned long long* d_cnt = nullptr;
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_side = nullptr, *d_late = nullptr, *d_flag = nullptr, *d_vflag = nullptr;
  u64* d_handles = nullptr;
  i64* d_ts = nullptr;
  PjEmit e{};
  JwPool pool{}, pool2{};  // ordered mode: the queue, and the one the next flush writes
  u64 nq = 0;              // entries in `pool`
  int slot_bits = 1;
  u64 kmax = 1;                        // entries one value can add: min(ceil(length / offset), max_windows_per_key)
  u64 n_store = 0, dead = 0;           // entries in the store, and how many of them are dead
  u64 n_vals = 0;                      // value slots in use (live and dead) since the last compaction
  u64 n_rec = 0, n_meta = 0, n_stage = 0;  // stage records, meta rows and staged handles since the last advance / eof
  SortScratch srt;                     // pool sort, ordering and compaction scratch
  PjOrdered o{};                       // advance / eof: the events in the reference's order
  u64* d_off = nullptr;                // the exclusive scan of their row counts
  u64 *d_vlive = nullptr, *d_vmap = nullptr;  // value compaction: live flags and their scan
  PjRows rows{};                       // the expanded rows
  u64 rows_cap = 0;
  HostCols hd[2];                      // down: key, window id, h0, h1, h2 | h3, mask, epoch
  HostCols hm, hl;                     // meta: key, window id, epoch; late: key, window id, epoch, activation, row
  std::vector<u64> late_rank;          // the late rows' source ranks: all zeros (one GPU)
  std::vector<u64> released;           // since the last advance / eof
  std::vector<u64> released_out;       // what the last advance / eof handed out
  bool undrained = false;     // a call whose counts are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
};

static const char* jwin_what(const bw_pjwin*) { return "windowed product join"; }
static const char* jwin_full_windows(const bw_pjwin*) { return " a key needs more than max_windows_per_key open windows;"; }
static const char* jwin_full_emit(const bw_pjwin*) { return " more than max_emit_rows emissions or meta rows since the last advance;"; }
static u64 jwin_counters(const bw_pjwin*) { return 10; }

bw_status bw_pjwin_create(bw_ctx* ctx, const bw_pjwin_spec* spec, bw_pjwin** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_pjwin_create: NULL argument");
  if (spec->struct_size != sizeof(bw_pjwin_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_pjwin_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed product joins run on one GPU (world == 1)");
  if (spec->emit_mode < BW_JOIN_EMIT_COMPLETE || spec->emit_mode > BW_JOIN_EMIT_RUNNING) CTX_FAIL(ctx, BW_ERR_SPEC, "bad emit_mode");
  if (spec->ordered != 0 && spec->ordered != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "ordered must be 0 or 1");
  if (spec->sides < 1 || spec->sides > BW_JW_MAXSIDES) CTX_FAIL(ctx, BW_ERR_SPEC, "sides must be in 1..%d", BW_JW_MAXSIDES);
  if (spec->max_windows_per_key < 1 || spec->max_windows_per_key > BW_JW_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_windows_per_key must be in 1..%d", BW_JW_MAXM);
  if (spec->length_us <= 0 || spec->length_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "length_us must be in 1..UTC_MAX - UTC_MIN");
  if (spec->offset_us <= 0 || spec->offset_us > spec->length_us) CTX_FAIL(ctx, BW_ERR_SPEC, "offset_us must be in 1..length_us");
  if (spec->align_us < BW_UTC_MIN_US || spec->align_us > BW_UTC_MAX_US) CTX_FAIL(ctx, BW_ERR_SPEC, "align_us out of range");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_queued_rows >= (1ULL << 31) - spec->max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "max_queued_rows + max_batch_rows must stay below 2^31");
  if (spec->max_emit_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "max_emit_rows must be below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_pjwin, void (*)(bw_pjwin*)> jp(new bw_pjwin(), bw_pjwin_destroy);  // torn down on every failure
  bw_pjwin* j = jp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_windows_per_key;
  const u64 per = (u64)((spec->length_us - 1) / spec->offset_us) + 1;
  j->kmax = std::min<u64>(per, (u64)M);
  PjTable& t = j->t;
  t.j.cap = cap;
  t.j.M = M;
  t.j.sides = spec->sides;
  while ((1ULL << j->slot_bits) < cap + 1) ++j->slot_bits;
  const u64 cells = (cap + 1) * (u64)M;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.j.keys, cap + 1));
  CU(ctx, own.dev(&t.j.st, cap + 1));
  CU(ctx, own.dev(&t.win, cells));
  CU(ctx, own.dev(&t.cell, cells));
  CU(ctx, own.dev(&t.rec_ord, cells));
  CU(ctx, own.dev(&t.rec_c, cells));
  CU(ctx, own.dev(&t.close_ord, cells));
  CU(ctx, own.dev(&t.j.err, 2));
  t.j.why = t.j.err + 1;
  t.err = t.j.err;
  t.why = t.j.why;
  CU(ctx, own.dev(&j->d_cnt, 10));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 80, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 16));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  const u64 q = spec->ordered ? spec->max_queued_rows : 0;
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_side, n));
  CU(ctx, own.dev(&j->d_late, n));
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_ts, n));
  if (spec->ordered) {
    if ((st = jwin_pool_alloc(ctx, own, j->pool, q + n)) != BW_OK) return st;
    if ((st = jwin_pool_alloc(ctx, own, j->pool2, q + n)) != BW_OK) return st;
  }
  PjEmit& e = j->e;
  for (u64** c : {&e.key, &e.wid, &e.epoch, &e.ord, &e.seq, &e.rec, &e.m_key, &e.m_wid, &e.m_epoch, &e.m_ord, &e.m_seq}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  for (u32** c : {&e.lo, &e.hi, &e.rb, &e.rn}) CU(ctx, own.dev(c, 4 * m));
  CU(ctx, own.dev(&e.rbase, 4 * m));
  PjOrdered& o = j->o;
  for (u64** c : {&o.cnt, &o.key, &o.wid, &o.epoch}) CU(ctx, own.dev(c, m + 1));
  CU(ctx, own.dev(&o.base, 4 * m));
  CU(ctx, own.dev(&o.len, 4 * m));
  CU(ctx, own.dev(&j->d_off, m + 1));
  // the store, the values, the staging buffer, the release buffer and the output grow with what the join holds and
  // emits (pjwin_room, pjwin_collect); they start at one batch
  PjStore& es = j->es;
  es.c.cap = n;
  CU(ctx, own.dev(&es.c.ref, n));
  CU(ctx, own.dev(&es.c.rank, n));
  CU(ctx, own.dev(&es.c.h, n));
  CU(ctx, own.dev(&es.vi, n));
  CU(ctx, own.dev(&j->d_flag, n));
  es.vcap = n;
  CU(ctx, own.dev(&es.vcnt, n));
  CU(ctx, own.dev(&j->d_vlive, n));
  CU(ctx, own.dev(&j->d_vmap, n));
  CU(ctx, own.dev(&j->d_vflag, n));
  e.max_stage = n;
  CU(ctx, own.dev(&e.stage, n));
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.max_queue = q;
  e.n_rows = j->d_cnt;
  e.n_meta = j->d_cnt + 1;
  e.n_late = j->d_cnt + 2;
  e.n_rel = j->d_cnt + 3;
  e.n_next = j->d_cnt + 4;
  e.n_rec = j->d_cnt + 5;
  e.n_stage = j->d_cnt + 6;
  es.c.n = j->d_cnt + 7;
  es.nv = j->d_cnt + 8;
  es.n_dead = j->d_cnt + 9;
  const u64 ns = std::max(std::max(m, l), q + n);
  CU(ctx, j->srt.reserve(own, ns, ns, j->s));
  size_t b = 0;
  CU(ctx, cub::DeviceScan::ExclusiveScan(nullptr, b, o.cnt, j->d_off, PjSatAdd{}, (u64)0, (int)(m + 1), j->s));
  CU(ctx, j->srt.grow_cub(own, b + 256));
  CU(ctx, j->hm.reserve(own, m, m));
  CU(ctx, j->hl.reserve(own, l, l));
  k_pjwin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = jp.release();
  return BW_OK;
}

void bw_pjwin_destroy(bw_pjwin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static JwParams pjwin_params(bw_pjwin* j, u64 epoch) {
  JwParams p{};
  p.emit_mode = j->spec.emit_mode;
  p.ordered = j->spec.ordered;
  p.length = j->spec.length_us;
  p.offset = j->spec.offset_us;
  p.align = j->spec.align_us;
  p.wait = j->spec.wait_us;
  p.now = j->now;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.batch_no = j->batch_no;
  return p;
}

// K8's drain (failure, released handles, queue count), then the counts only this join keeps
static bw_status pjwin_drain(bw_pjwin* j) {
  const bool pending = j->undrained;
  bw_status st = jwin_drain(j);
  if (st != BW_OK || !pending) return st;
  j->n_meta = j->h_cnt[1];
  j->n_rec = j->h_cnt[5];
  j->n_stage = j->h_cnt[6];
  j->n_store = j->h_cnt[7];
  j->n_vals = j->h_cnt[8];
  j->dead += j->h_cnt[9];
  CU(j->ctx, cudaMemsetAsync(j->d_cnt + 9, 0, 8, j->s));
  return BW_OK;
}

// Before a call that can play `rows` values (and ordered the queued entries): compact the store and the values once dead
// entries outnumber live ones, then grow the store, the values, the staging buffer and the release buffer so that
// nothing the call can add, stage or release overflows them.  Called after the drain: nothing on the stream reads them.
static bw_status pjwin_room(bw_pjwin* j, u64 rows) {
  bw_ctx* ctx = j->ctx;
  bw_status st = jwin_room(j, rows);
  if (st != BW_OK) return st;
  PjStore& es = j->es;
  PjEmit& e = j->e;
  const u64 vadds = rows + (j->spec.ordered ? j->nq : 0), adds = vadds * j->kmax;
  if (j->dead && j->dead >= j->n_store - j->dead) {  // stream compaction of the values, then of the entries (both stable)
    const int grid = ctx->sm_count * 4;
    size_t b = 0, b2 = 0, b3 = 0;
    CU(ctx, cub::DeviceSelect::Flagged(nullptr, b, es.c.h, j->d_flag, es.c.n, (int64_t)j->n_store, j->s));
    CU(ctx, cub::DeviceSelect::Flagged(nullptr, b2, es.vcnt, j->d_vflag, es.nv, (int64_t)j->n_vals, j->s));
    CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b3, j->d_vlive, j->d_vmap, (int64_t)j->n_vals, j->s));
    CU(ctx, j->srt.grow_cub(j->own, std::max(std::max(b, b2), b3) + 256));
    size_t tb = j->srt.cub_bytes;
    if (j->n_vals) {
      k_pjwin_vlive<<<grid, 256, 0, j->s>>>(es.vcnt, j->d_vlive, j->d_vflag, j->n_vals);
      CU(ctx, cub::DeviceScan::ExclusiveSum(j->srt.cub, tb, j->d_vlive, j->d_vmap, (int64_t)j->n_vals, j->s));
      tb = j->srt.cub_bytes;
      CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.vcnt, j->d_vflag, es.nv, (int64_t)j->n_vals, j->s));
    }
    k_cwin_live<<<grid, 256, 0, j->s>>>(es.c.ref, j->d_flag, j->n_store);
    for (int c = 0; c < 4; ++c) {
      tb = j->srt.cub_bytes;
      if (c == 0) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.c.h, j->d_flag, es.c.n, (int64_t)j->n_store, j->s));
      if (c == 1) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.c.rank, j->d_flag, es.c.n, (int64_t)j->n_store, j->s));
      if (c == 2) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.vi, j->d_flag, es.c.n, (int64_t)j->n_store, j->s));
      if (c == 3) CU(ctx, cub::DeviceSelect::Flagged(j->srt.cub, tb, es.c.ref, j->d_flag, es.c.n, (int64_t)j->n_store, j->s));
    }
    j->n_store -= j->dead;
    j->dead = 0;
    if (j->n_vals && j->n_store) k_pjwin_remap<<<grid, 256, 0, j->s>>>(es.vi, j->d_vmap, j->n_store);
    CU(ctx, cudaGetLastError());
    CU(ctx, cudaMemcpyAsync(j->h_cnt + 8, es.nv, 8, cudaMemcpyDeviceToHost, j->s));
    CU(ctx, cudaStreamSynchronize(j->s));
    j->n_vals = j->n_vals ? j->h_cnt[8] : 0;
  }
  const u64 live = j->n_store - j->dead;
  if (j->n_store + adds > es.c.cap) {
    const u64 grow = std::max<u64>(j->n_store + adds, 2 * es.c.cap);
    es.c.cap = 0;  // (a failed regrow leaves the store unusable: the next call fails here again)
    CU(ctx, collect_grow_keep(j, &es.c.ref, j->n_store, grow));
    CU(ctx, collect_grow_keep(j, &es.c.rank, j->n_store, grow));
    CU(ctx, collect_grow_keep(j, &es.c.h, j->n_store, grow));
    CU(ctx, collect_grow_keep(j, &es.vi, j->n_store, grow));
    CU(ctx, j->own.regrow(Owner::DEV, &j->d_flag, grow));
    es.c.cap = grow;
  }
  if (j->n_vals + vadds > es.vcap) {
    const u64 grow = std::max<u64>(j->n_vals + vadds, 2 * es.vcap);
    es.vcap = 0;
    CU(ctx, collect_grow_keep(j, &es.vcnt, j->n_vals, grow));
    CU(ctx, j->own.regrow(Owner::DEV, &j->d_vlive, grow));
    CU(ctx, j->own.regrow(Owner::DEV, &j->d_vmap, grow));
    CU(ctx, j->own.regrow(Owner::DEV, &j->d_vflag, grow));
    es.vcap = grow;
  }
  if (j->n_stage + live + adds > e.max_stage) {
    const u64 grow = std::max<u64>(j->n_stage + live + adds, 2 * e.max_stage);
    e.max_stage = 0;
    CU(ctx, collect_grow_keep(j, &e.stage, j->n_stage, grow));
    e.max_stage = grow;
  }
  return BW_OK;
}

#define PJWIN_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "windowed product join: an earlier call failed on the device; the join is unusable")

// after the per-key kernels of a call: stage the emitting windows' lists, kill dead entries, release (k_pjwin_gather)
static bw_status pjwin_gather(bw_pjwin* j, const JwParams& p) {
  k_pjwin_gather<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->n_rec, j->n_meta);
  CU(j->ctx, cudaGetLastError());
  return BW_OK;
}

// ordered mode: sort the pool's due entries into play order (K8's sort); then flush every woken key (k_pjwin_flush)
static bw_status pjwin_flush(bw_pjwin* j, const JwParams& p, u64 n) {
  bw_ctx* ctx = j->ctx;
  bw_status st = j->spec.ordered ? jwin_sort_pool(j, j->t.j, p, n) : BW_OK;
  if (st != BW_OK) return st;
  PjEmit e = j->e;
  e.next = j->pool2;
  k_pjwin_flush<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, j->es, p, j->pool, j->srt.perm);
  CU(ctx, cudaGetLastError());
  if (j->spec.ordered) std::swap(j->pool, j->pool2);  // the next call reads what this flush carried over (count: jwin_drain)
  return pjwin_gather(j, p);
}

bw_status bw_pjwin_apply_device(bw_pjwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles, const int64_t* d_ts_us,
                                uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  PJWIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed product join: rows > max_batch_rows");
  if (rows && (!d_keys || !d_side || !d_handles || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "windowed product join: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "windowed product join: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = pjwin_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = pjwin_params(j, epoch);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = pjwin_room(j, rows)) != BW_OK) return st;
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_pjwin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted, j->k.d_head,
                                                     d_handles, d_side, d_ts_us, j->d_late, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return pjwin_flush(j, p, j->nq + rows);
  return pjwin_gather(j, p);
}

static bw_status pjwin_apply_device_fn(bw_pjwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles,
                                       const int64_t* d_ts_us, uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  bw_status st = bw_pjwin_apply_device(j, d_keys, d_side, d_handles, d_ts_us, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  return pjwin_drain(j);  // (jwin_apply_host drains once more: then nothing is pending)
}

bw_status bw_pjwin_apply(bw_pjwin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us, uint64_t rows,
                         uint64_t epoch, int64_t system_now_us) {
  if (j) {
    PJWIN_REFUSE_FAILED(j);
    bw_status st = pjwin_drain(j);  // (before jwin_apply_host's own drain, which would skip this join's counts)
    if (st != BW_OK) return st;
  }
  return jwin_apply_host(j, keys, side, handles, ts_us, rows, epoch, system_now_us, pjwin_apply_device_fn);
}

// advance / eof: the events in the reference's order (order_perm), their row counts and the saturating scan of them;
// the host grows the output to the total; k_pjwin_expand writes every row in that order
static bw_status pjwin_expand(bw_pjwin* j, u64 nd, u64* total) {
  bw_ctx* ctx = j->ctx;
  *total = 0;
  if (!nd) return BW_OK;
  SortScratch& x = j->srt;
  bw_status st = order_perm(ctx, x, j->s, nd, j->e.key, j->e.seq, j->e.ord, nullptr, std::max<u64>(j->calls - j->first_call, 1), j->first_call,
                            nullptr);
  if (st != BW_OK) return st;
  const int grid = ctx->sm_count * 4;
  PjOrdered o = j->o;
  k_pjwin_count<<<grid, 256, 0, j->s>>>(j->e, o, j->spec.sides, x.perm, nd);
  CU(ctx, cudaMemsetAsync(o.cnt + nd, 0, 8, j->s));
  size_t tb = x.cub_bytes;
  CU(ctx, cub::DeviceScan::ExclusiveScan(x.cub, tb, o.cnt, j->d_off, PjSatAdd{}, (u64)0, (int)(nd + 1), j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt + 12, j->d_off + nd, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 n = j->h_cnt[12];
  if (n > j->spec.max_product_rows) {
    j->failed = true;
    CTX_FAIL(ctx, BW_ERR_CAPACITY, "windowed product join ran out of capacity: %llu product rows since the last advance, more than "
             "max_product_rows (%llu)", (unsigned long long)n, (unsigned long long)j->spec.max_product_rows);
  }
  if (n > j->rows_cap) {
    j->rows_cap = 0;
    for (u64** c : {&j->rows.key, &j->rows.wid, &j->rows.h0, &j->rows.h1, &j->rows.h2, &j->rows.h3, &j->rows.mask, &j->rows.epoch})
      CU(ctx, j->own.regrow(Owner::DEV, c, n));
    j->rows_cap = n;
  }
  CU(ctx, j->hd[0].reserve(j->own, n, n));
  CU(ctx, j->hd[1].reserve(j->own, n, n));
  k_pjwin_expand<<<ctx->sm_count * 8, 256, 0, j->s>>>(o, j->d_off, nd, j->spec.sides, j->e.stage, j->rows, n);
  const u64* src[] = {j->rows.key, j->rows.wid, j->rows.h0, j->rows.h1, j->rows.h2, j->rows.h3, j->rows.mask, j->rows.epoch};
  for (int c = 0; c < 8; ++c) CU(ctx, cudaMemcpyAsync(j->hd[c / 5].col[c % 5], src[c], n * 8, cudaMemcpyDeviceToHost, j->s));
  *total = n;
  return BW_OK;
}

static bw_status pjwin_collect(bw_pjwin* j, bw_jwin_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = pjwin_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 24, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 nd = j->h_cnt[0], nm = j->h_cnt[1], nl = j->h_cnt[2];  // all within bounds: jwin_drain passed
  u64 n = 0;
  if ((st = pjwin_expand(j, nd, &n)) != BW_OK) return st;
  const PjEmit& e = j->e;
  const u64* meta[] = {e.m_key, e.m_wid, e.m_epoch};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(j, nm, e.m_key, e.m_seq, e.m_ord, meta, 3, &j->hm)) != BW_OK) return st;
  if ((st = jwin_ship(j, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &j->hl)) != BW_OK) return st;
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 24, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 5, 0, 16, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->n_rec = j->n_meta = j->n_stage = 0;
  j->first_call = j->calls;
  out->n_down = n;
  out->down_key = j->hd[0].col[0];
  out->down_window_id = (const int64_t*)j->hd[0].col[1];
  out->down_handle[0] = j->hd[0].col[2];
  out->down_handle[1] = j->hd[0].col[3];
  out->down_handle[2] = j->hd[0].col[4];
  out->down_handle[3] = j->hd[1].col[0];
  out->down_mask = j->hd[1].col[1];
  out->down_epoch = j->hd[1].col[2];
  out->n_meta = nm;
  out->meta_key = j->hm.col[0];
  out->meta_window_id = (const int64_t*)j->hm.col[1];
  out->meta_epoch = j->hm.col[2];
  out->n_late = nl;
  out->late_key = j->hl.col[0];
  out->late_window_id = (const int64_t*)j->hl.col[1];
  out->late_epoch = j->hl.col[2];
  out->late_activation = j->hl.col[3];
  out->late_row = j->hl.col[4];
  j->late_rank.assign(nl, 0);
  out->late_rank = j->late_rank.data();
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys (K8's k_jwin_mark), then flush them (ordered: through the pool)
static bw_status pjwin_wake(bw_pjwin* j, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = pjwin_drain(j);
  if (st != BW_OK) return st;
  if ((st = pjwin_room(j, 0)) != BW_OK) return st;
  const JwParams p = pjwin_params(j, j->last_epoch);
  k_jwin_mark<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t.j, j->t.win, p, eof);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return pjwin_flush(j, p, j->nq);
}

bw_status bw_pjwin_advance(bw_pjwin* j, int64_t system_now_us, bw_jwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  PJWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > j->now) j->now = system_now_us;
    bw_status st = pjwin_wake(j, 0);
    if (st != BW_OK) return st;
  }
  return pjwin_collect(j, out);
}

bw_status bw_pjwin_eof(bw_pjwin* j, bw_jwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  PJWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = pjwin_wake(j, 1);
  if (st != BW_OK) return st;
  return pjwin_collect(j, out);
}

// ===========================================================================
// K15 host side: keyed join (bw_kjoin.cuh)
// ===========================================================================
struct bw_kjoin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_kjoin_spec spec{};
  KjTable t{};
  CwStore es{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;  // err, why
  // events, released, stage records, staged, store entries, dead entries, killed entries
  unsigned long long* d_cnt = nullptr;
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_side = nullptr, *d_flag = nullptr;
  u64* d_handles = nullptr;
  KjEmit e{};
  u64 n_store = 0, dead = 0;   // entries in the store, and how many of them are dead
  u64 n_rec = 0, n_stage = 0;  // stage records and staged handles since the last advance / eof
  SortScratch srt;             // ordering and compaction scratch
  PjOrdered o{};               // advance / eof: the events in the reference's order
  u64* d_off = nullptr;        // the exclusive scan of their row counts
  u64* d_zero = nullptr;       // the window-id column K14's count kernel reads: zeros
  PjRows rows{};               // the expanded rows (its window-id column is not copied out)
  u64 rows_cap = 0;
  HostCols hd[2];              // key, h0, h1, h2, h3 | mask, epoch
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;         // a call whose counts are not read back yet
  u64 outstanding = 0;            // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  bool failed = false;
};

bw_status bw_kjoin_create(bw_ctx* ctx, const bw_kjoin_spec* spec, bw_kjoin** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_kjoin_create: NULL argument");
  if (spec->struct_size != sizeof(bw_kjoin_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_kjoin_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed joins run on one GPU (world == 1)");
  if (spec->insert_mode < BW_JOIN_INSERT_FIRST || spec->insert_mode > BW_JOIN_INSERT_PRODUCT) CTX_FAIL(ctx, BW_ERR_SPEC, "bad insert_mode");
  if (spec->emit_mode < BW_JOIN_EMIT_COMPLETE || spec->emit_mode > BW_JOIN_EMIT_RUNNING) CTX_FAIL(ctx, BW_ERR_SPEC, "bad emit_mode");
  if (spec->sides < 1 || spec->sides > BW_JW_MAXSIDES) CTX_FAIL(ctx, BW_ERR_SPEC, "sides must be in 1..%d", BW_JW_MAXSIDES);
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_emit_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "max_emit_rows must be below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_kjoin, void (*)(bw_kjoin*)> jp(new bw_kjoin(), bw_kjoin_destroy);  // torn down on every failure
  bw_kjoin* j = jp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  KjTable& t = j->t;
  t.cap = cap;
  t.sides = spec->sides;
  t.insert_mode = spec->insert_mode;
  t.emit_mode = spec->emit_mode;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.keys, cap + 1));
  CU(ctx, own.dev(&t.cell, cap + 1));
  CU(ctx, own.dev(&t.live, cap + 1));
  CU(ctx, own.dev(&t.rec_ord, cap + 1));
  CU(ctx, own.dev(&t.rec_c, cap + 1));
  CU(ctx, own.dev(&t.err, 2));
  t.why = t.err + 1;
  CU(ctx, own.dev(&j->d_cnt, 7));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 56, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 16));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1);
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_side, n));
  CU(ctx, own.dev(&j->d_handles, n));
  KjEmit& e = j->e;
  for (u64** c : {&e.key, &e.epoch, &e.ord, &e.seq, &e.rec}) CU(ctx, own.dev(c, m));
  for (u32** c : {&e.lo, &e.hi, &e.rb, &e.rn}) CU(ctx, own.dev(c, 4 * m));
  CU(ctx, own.dev(&e.rbase, 4 * m));
  PjOrdered& o = j->o;
  for (u64** c : {&o.cnt, &o.key, &o.wid, &o.epoch}) CU(ctx, own.dev(c, m + 1));
  CU(ctx, own.dev(&o.base, 4 * m));
  CU(ctx, own.dev(&o.len, 4 * m));
  CU(ctx, own.dev(&j->d_off, m + 1));
  CU(ctx, own.dev(&j->d_zero, m));
  CU(ctx, cudaMemsetAsync(j->d_zero, 0, m * 8, j->s));
  // the store, the staging buffer, the release buffer and the output grow with what the join holds and emits
  // (store_room, jwin_room, kjoin_expand); they start at one batch
  CwStore& es = j->es;
  es.cap = n;
  CU(ctx, own.dev(&es.ref, n));
  CU(ctx, own.dev(&es.rank, n));
  CU(ctx, own.dev(&es.h, n));
  CU(ctx, own.dev(&j->d_flag, n));
  e.max_stage = n;
  CU(ctx, own.dev(&e.stage, n));
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.n_rows = j->d_cnt;
  e.n_rel = j->d_cnt + 1;
  e.n_rec = j->d_cnt + 2;
  e.n_stage = j->d_cnt + 3;
  es.n = j->d_cnt + 4;
  e.n_kill = j->d_cnt + 6;
  CU(ctx, j->srt.reserve(own, m, m, j->s));
  size_t b = 0;
  CU(ctx, cub::DeviceScan::ExclusiveScan(nullptr, b, o.cnt, j->d_off, PjSatAdd{}, (u64)0, (int)(m + 1), j->s));
  CU(ctx, j->srt.grow_cub(own, b + 256));
  k_kjoin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = jp.release();
  return BW_OK;
}

void bw_kjoin_destroy(bw_kjoin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static KjParams kjoin_params(bw_kjoin* j, u64 epoch, int eof) {
  KjParams p;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.eof = eof;
  return p;
}

#define KJOIN_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "keyed join: an earlier call failed on the device; the join is unusable")

// wait for the last call; fail on a device-side overflow or a bad side; then take its released handles and its counts,
// so the device buffer only ever holds one call's releases
static bw_status kjoin_drain(bw_kjoin* j) {
  bw_ctx* ctx = j->ctx;
  KJOIN_REFUSE_FAILED(j);
  if (!j->undrained) return BW_OK;
  CU(ctx, cudaMemcpyAsync(j->h_err, j->t.err, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 56, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  if (j->h_err[0]) {
    j->failed = true;
    const u32 w = j->h_err[1];
    CTX_FAIL(ctx, (bw_status)j->h_err[0], "keyed join kernel %s:%s%s%s%s%s%s",
             j->h_err[0] == BW_ERR_SPEC ? "rejected its input" : "ran out of capacity",
             w & BW_JW_BAD_SIDE ? " a side column value is not below sides;" : "", w & BW_JW_FULL_TABLE ? " key table full (raise capacity_hint);" : "",
             w & BW_JW_FULL_EMIT ? " more than max_emit_rows emissions since the last advance;" : "",
             w & BW_CW_FULL_STORE ? " entry store or staging buffer full;" : "",
             w & BW_PJ_FULL_SIDE ? " a key's side list reached 2^32 values;" : "", w ? "" : " (no reason recorded)");
  }
  const u64 nr = j->h_cnt[1];
  j->outstanding -= std::min(nr, j->outstanding);
  if (nr) {
    const size_t at = j->released.size();
    j->released.resize(at + nr);
    CU(ctx, cudaMemcpyAsync(j->released.data() + at, j->e.rel, nr * 8, cudaMemcpyDeviceToHost, j->s));
  }
  j->n_rec = j->h_cnt[2];
  j->n_stage = j->h_cnt[3];
  j->n_store = j->h_cnt[4];
  j->dead += j->h_cnt[5];
  CU(ctx, cudaMemsetAsync(j->d_cnt + 5, 0, 16, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 1, 0, 8, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->undrained = false;
  return BW_OK;
}

// after the per-key kernel of a call: stage the emitting keys' lists, kill dead entries, release (k_kjoin_gather)
static bw_status kjoin_gather(bw_kjoin* j, const KjParams& p) {
  k_kjoin_gather<<<j->ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->n_rec, j->d_cnt + 5);
  CU(j->ctx, cudaGetLastError());
  return BW_OK;
}

bw_status bw_kjoin_apply_device(bw_kjoin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles, uint64_t rows,
                                uint64_t epoch) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  KJOIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed join: rows > max_batch_rows");
  if (rows && (!d_keys || !d_side || !d_handles)) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed join: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "keyed join: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = kjoin_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  const KjParams p = kjoin_params(j, epoch, 0);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = jwin_room(j, rows)) != BW_OK) return st;
  if ((st = store_room(j, rows)) != BW_OK) return st;  // (a value adds at most one entry)
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_kjoin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, j->es, p, j->k.d_ksorted, j->k.d_isorted, j->k.d_head, d_handles, d_side,
                                                     rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return kjoin_gather(j, p);
}

bw_status bw_kjoin_apply(bw_kjoin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, uint64_t rows, uint64_t epoch) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  KJOIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed join: rows > max_batch_rows");
  if (rows && (!keys || !side || !handles)) CTX_FAIL(ctx, BW_ERR_SPEC, "keyed join: NULL column");
  for (u64 i = 0; i < rows; ++i)
    if (side[i] >= (u32)j->spec.sides)
      CTX_FAIL(ctx, BW_ERR_SPEC, "keyed join: side %u of row %llu is not below sides", side[i], (unsigned long long)i);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = kjoin_drain(j);
  if (st != BW_OK) return st;
  if (rows) {
    CU(ctx, cudaMemcpyAsync(j->k.d_keys, keys, rows * 8, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_side, side, rows, cudaMemcpyHostToDevice, j->s));
    CU(ctx, cudaMemcpyAsync(j->d_handles, handles, rows * 8, cudaMemcpyHostToDevice, j->s));
  }
  st = bw_kjoin_apply_device(j, j->k.d_keys, j->d_side, j->d_handles, rows, epoch);
  if (st != BW_OK) return st;
  // the host columns may be reused by the caller once this returns
  return kjoin_drain(j);
}

// advance / eof: the events in the reference's order (order_perm), their row counts and the saturating scan of them
// (K14's k_pjwin_count, over a zero window-id column); the host grows the output to the total; K14's k_pjwin_expand
// writes every row in that order
static bw_status kjoin_expand(bw_kjoin* j, u64 nd, u64* total) {
  bw_ctx* ctx = j->ctx;
  *total = 0;
  if (!nd) return BW_OK;
  SortScratch& x = j->srt;
  const KjEmit& e = j->e;
  bw_status st = order_perm(ctx, x, j->s, nd, e.key, e.seq, e.ord, nullptr, std::max<u64>(j->calls - j->first_call, 1), j->first_call,
                            nullptr);
  if (st != BW_OK) return st;
  PjEmit v{};  // the event columns as K14 lays them out
  v.key = e.key;
  v.wid = j->d_zero;
  v.epoch = e.epoch;
  v.rec = e.rec;
  v.lo = e.lo;
  v.hi = e.hi;
  v.rb = e.rb;
  v.rn = e.rn;
  v.rbase = e.rbase;
  const PjOrdered o = j->o;
  k_pjwin_count<<<ctx->sm_count * 4, 256, 0, j->s>>>(v, o, j->spec.sides, x.perm, nd);
  CU(ctx, cudaMemsetAsync(o.cnt + nd, 0, 8, j->s));
  size_t tb = x.cub_bytes;
  CU(ctx, cub::DeviceScan::ExclusiveScan(x.cub, tb, o.cnt, j->d_off, PjSatAdd{}, (u64)0, (int)(nd + 1), j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt + 8, j->d_off + nd, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 n = j->h_cnt[8];
  if (n > j->spec.max_product_rows) {
    j->failed = true;
    CTX_FAIL(ctx, BW_ERR_CAPACITY, "keyed join ran out of capacity: %llu product rows since the last advance, more than max_product_rows "
             "(%llu)", (unsigned long long)n, (unsigned long long)j->spec.max_product_rows);
  }
  if (n > j->rows_cap) {
    j->rows_cap = 0;
    for (u64** c : {&j->rows.key, &j->rows.wid, &j->rows.h0, &j->rows.h1, &j->rows.h2, &j->rows.h3, &j->rows.mask, &j->rows.epoch})
      CU(ctx, j->own.regrow(Owner::DEV, c, n));
    j->rows_cap = n;
  }
  CU(ctx, j->hd[0].reserve(j->own, n, n));
  CU(ctx, j->hd[1].reserve(j->own, n, n));
  k_pjwin_expand<<<ctx->sm_count * 8, 256, 0, j->s>>>(o, j->d_off, nd, j->spec.sides, e.stage, j->rows, n);
  const u64* src[] = {j->rows.key, j->rows.h0, j->rows.h1, j->rows.h2, j->rows.h3, j->rows.mask, j->rows.epoch};
  for (int c = 0; c < 7; ++c) CU(ctx, cudaMemcpyAsync(j->hd[c / 5].col[c % 5], src[c], n * 8, cudaMemcpyDeviceToHost, j->s));
  *total = n;
  return BW_OK;
}

static bw_status kjoin_collect(bw_kjoin* j, bw_kjoin_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = kjoin_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 nd = j->h_cnt[0];  // within bounds: kjoin_drain passed
  u64 n = 0;
  if ((st = kjoin_expand(j, nd, &n)) != BW_OK) return st;
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 2, 0, 16, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->n_rec = j->n_stage = 0;
  j->first_call = j->calls;
  out->n = n;
  out->key = j->hd[0].col[0];
  for (int s = 0; s < 4; ++s) out->handle[s] = j->hd[0].col[1 + s];
  out->mask = j->hd[1].col[0];
  out->epoch = j->hd[1].col[1];
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

bw_status bw_kjoin_advance(bw_kjoin* j, bw_kjoin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  KJOIN_REFUSE_FAILED(j);
  CU(j->ctx, cudaSetDevice(j->ctx->device));
  return kjoin_collect(j, out);
}

bw_status bw_kjoin_eof(bw_kjoin* j, bw_kjoin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  KJOIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = kjoin_drain(j);
  if (st != BW_OK) return st;
  if ((st = store_room(j, 0)) != BW_OK) return st;  // (staging for every entry held)
  const KjParams p = kjoin_params(j, j->last_epoch, 1);
  k_kjoin_eof<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, j->e, p);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if ((st = kjoin_gather(j, p)) != BW_OK) return st;
  return kjoin_collect(j, out);
}

// ===========================================================================
// K16 host side: windowed product join over session windows (bw_spjwin.cuh)
// ===========================================================================
// K9's store growth and compaction (store_room), K8's drain, release-buffer growth and pool sort (jwin_drain, jwin_room,
// jwin_sort_pool, jwin_ship) and K14's expansion read these members by the names bw_pjwin / bw_kjoin give them.
struct bw_spjwin {
  Owner own;  // every buffer and the stream below
  bw_ctx* ctx = nullptr;
  bw_spjwin_spec spec{};
  SpTable t{};
  CwStore es{};
  KeyedScratch k;
  cudaStream_t s = nullptr;
  u32* h_err = nullptr;  // err, why
  // events, meta, late, released, carried-over queue entries, stage records, staged, store entries, dead entries, merged
  // ids, merges
  unsigned long long* d_cnt = nullptr;
  unsigned long long* h_cnt = nullptr;
  unsigned char *d_side = nullptr, *d_late = nullptr, *d_flag = nullptr;
  u64* d_handles = nullptr;
  i64* d_ts = nullptr;
  SpEmit e{};
  JwPool pool{}, pool2{};  // ordered mode: the queue, and the one the next flush writes
  u64 nq = 0;              // entries in `pool`
  int slot_bits = 1;
  u64 n_store = 0, dead = 0;               // entries in the store, and how many of them are dead
  u64 n_rec = 0, n_meta = 0, n_stage = 0;  // stage records, meta rows and staged handles since the last advance / eof
  u64 n_mrg = 0;                           // keys that merged, so far
  SortScratch srt;                         // pool sort, ordering and compaction scratch
  PjOrdered o{};                           // advance / eof: the events in the reference's order
  u64* d_off = nullptr;                    // the exclusive scan of their row counts
  PjRows rows{};                           // the expanded rows
  u64 rows_cap = 0;
  HostCols hd[2];  // down: key, window id, h0, h1, h2 | h3, mask, epoch
  HostCols hm[2];  // meta: key, window id, open, close, epoch | merged count, merged offset
  HostCols hl;     // late: key, window id, epoch, activation, row
  i64* h_mids = nullptr;
  std::vector<u64> merged_off;
  std::vector<i64> merged_ids;
  std::vector<u64> released;      // since the last advance / eof
  std::vector<u64> released_out;  // what the last advance / eof handed out
  bool undrained = false;     // a call whose counts are not read back yet
  u64 outstanding = 0;        // handles passed in and not released yet: what the next call can release, besides its own
  u32 batch_no = 0;
  u64 calls = 0, first_call = 0;  // calls (activations, notify phases, EOF) so far; the first not yet collected
  u64 last_epoch = 0;
  i64 now = INT64_MIN;
  bool failed = false;
};

static const char* jwin_what(const bw_spjwin*) { return "session product join"; }
static const char* jwin_full_windows(const bw_spjwin*) { return " a key needs more than max_sessions_per_key sessions or merged ids;"; }
static const char* jwin_full_emit(const bw_spjwin*) {
  return " more than max_emit_rows emissions, meta rows or merged ids since the last advance;";
}
static u64 jwin_counters(const bw_spjwin*) { return 11; }

bw_status bw_spjwin_create(bw_ctx* ctx, const bw_spjwin_spec* spec, bw_spjwin** out) {
  if (!ctx || !spec || !out) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_spjwin_create: NULL argument");
  if (spec->struct_size != sizeof(bw_spjwin_spec)) CTX_FAIL(ctx, BW_ERR_SPEC, "bw_spjwin_spec.struct_size mismatch");
  if (ctx->world != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "session product joins run on one GPU (world == 1)");
  if (spec->emit_mode < BW_JOIN_EMIT_COMPLETE || spec->emit_mode > BW_JOIN_EMIT_RUNNING) CTX_FAIL(ctx, BW_ERR_SPEC, "bad emit_mode");
  if (spec->ordered != 0 && spec->ordered != 1) CTX_FAIL(ctx, BW_ERR_SPEC, "ordered must be 0 or 1");
  if (spec->sides < 1 || spec->sides > BW_JW_MAXSIDES) CTX_FAIL(ctx, BW_ERR_SPEC, "sides must be in 1..%d", BW_JW_MAXSIDES);
  if (spec->max_sessions_per_key < 1 || spec->max_sessions_per_key > BW_SESS_MAXM)
    CTX_FAIL(ctx, BW_ERR_SPEC, "max_sessions_per_key must be in 1..%d", BW_SESS_MAXM);
  if (spec->gap_us < 0 || spec->gap_us > BW_UTC_MAX_US - BW_UTC_MIN_US) CTX_FAIL(ctx, BW_ERR_SPEC, "gap_us must be in 0..UTC_MAX - UTC_MIN");
  if (spec->wait_us < 0) CTX_FAIL(ctx, BW_ERR_SPEC, "wait_us must not be negative");
  if (spec->max_batch_rows == 0 || spec->max_batch_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "bad max_batch_rows");
  if (spec->max_queued_rows >= (1ULL << 31) - spec->max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "max_queued_rows + max_batch_rows must stay below 2^31");
  if (spec->max_emit_rows >= (1ULL << 31)) CTX_FAIL(ctx, BW_ERR_SPEC, "max_emit_rows must be below 2^31");
  if (spec->capacity_hint >= (1ULL << 30)) CTX_FAIL(ctx, BW_ERR_SPEC, "capacity_hint must be below 2^30");
  CU(ctx, cudaSetDevice(ctx->device));
  std::unique_ptr<bw_spjwin, void (*)(bw_spjwin*)> jp(new bw_spjwin(), bw_spjwin_destroy);  // torn down on every failure
  bw_spjwin* j = jp.get();
  Owner& own = j->own;
  j->ctx = ctx;
  j->spec = *spec;
  const u64 cap = std::max<u64>(1024, 2 * std::max<u64>(spec->capacity_hint, 1));
  const int M = spec->max_sessions_per_key;
  const u64 cells = (cap + 1) * (u64)M;
  SpTable& t = j->t;
  t.j.cap = cap;
  t.j.M = M;
  t.j.sides = spec->sides;
  t.gap = spec->gap_us;
  while ((1ULL << j->slot_bits) < cap + 1) ++j->slot_bits;
  CU(ctx, own.stream(&j->s));
  CU(ctx, own.dev(&t.j.keys, cap + 1));
  CU(ctx, own.dev(&t.j.st, cap + 1));
  CU(ctx, own.dev(&t.kx, cap + 1));
  CU(ctx, own.dev(&t.rec, cells));
  CU(ctx, own.dev(&t.mrg, 2 * cells));
  CU(ctx, own.dev(&t.cell, cells));
  CU(ctx, own.dev(&t.rec_ord, cells));
  CU(ctx, own.dev(&t.rec_c, cells));
  CU(ctx, own.dev(&t.close_ord, cells));
  CU(ctx, own.dev(&t.mord, cells));
  CU(ctx, own.dev(&t.hop, cells));
  t.j.win = nullptr;  // (K8's window records and K14's: sessions live in rec)
  t.win = nullptr;
  CU(ctx, own.dev(&t.j.err, 2));
  t.j.why = t.j.err + 1;
  t.err = t.j.err;
  t.why = t.j.why;
  CU(ctx, own.dev(&j->d_cnt, 11));
  CU(ctx, cudaMemsetAsync(t.err, 0, 8, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 88, j->s));
  CU(ctx, own.host(&j->h_err, 64 / sizeof(u32)));
  CU(ctx, own.host(&j->h_cnt, 16));
  const u64 n = spec->max_batch_rows, m = std::max<u64>(spec->max_emit_rows, 1), l = std::max<u64>(spec->max_late_rows, 1);
  const u64 q = spec->ordered ? spec->max_queued_rows : 0;
  bw_status st = keyed_alloc(ctx, own, j->k, n, j->s);
  if (st != BW_OK) return st;
  CU(ctx, own.dev(&j->d_side, n));
  CU(ctx, own.dev(&j->d_late, n));
  CU(ctx, own.dev(&j->d_handles, n));
  CU(ctx, own.dev(&j->d_ts, n));
  if (spec->ordered) {
    if ((st = jwin_pool_alloc(ctx, own, j->pool, q + n)) != BW_OK) return st;
    if ((st = jwin_pool_alloc(ctx, own, j->pool2, q + n)) != BW_OK) return st;
  }
  SpEmit& e = j->e;
  for (u64** c : {&e.key, &e.wid, &e.epoch, &e.ord, &e.seq, &e.rec, &e.m_key, &e.m_wid, &e.m_epoch, &e.m_ord, &e.m_seq, &e.m_moff, &e.m_mcnt})
    CU(ctx, own.dev(c, m));
  for (i64** c : {&e.m_open, &e.m_close, &e.mids}) CU(ctx, own.dev(c, m));
  for (u64** c : {&e.l_key, &e.l_wid, &e.l_epoch, &e.l_act, &e.l_row, &e.l_ord, &e.l_seq}) CU(ctx, own.dev(c, l));
  for (u32** c : {&e.lo, &e.hi, &e.rb, &e.rn}) CU(ctx, own.dev(c, 4 * m));
  CU(ctx, own.dev(&e.rbase, 4 * m));
  PjOrdered& o = j->o;
  for (u64** c : {&o.cnt, &o.key, &o.wid, &o.epoch}) CU(ctx, own.dev(c, m + 1));
  CU(ctx, own.dev(&o.base, 4 * m));
  CU(ctx, own.dev(&o.len, 4 * m));
  CU(ctx, own.dev(&j->d_off, m + 1));
  // the store, the staging buffer, the release buffer and the output grow with what the join holds and emits
  // (spjwin_room, spjwin_gather, spjwin_expand); they start at one batch
  CwStore& es = j->es;
  es.cap = n;
  CU(ctx, own.dev(&es.ref, n));
  CU(ctx, own.dev(&es.rank, n));
  CU(ctx, own.dev(&es.h, n));
  CU(ctx, own.dev(&j->d_flag, n));
  e.max_stage = n;
  CU(ctx, own.dev(&e.stage, n));
  e.max_rel = n;
  CU(ctx, own.dev(&e.rel, e.max_rel));
  e.max_rows = spec->max_emit_rows;
  e.max_late = spec->max_late_rows;
  e.max_queue = q;
  e.n_rows = j->d_cnt;
  e.n_meta = j->d_cnt + 1;
  e.n_late = j->d_cnt + 2;
  e.n_rel = j->d_cnt + 3;  // (jwin_drain reads these two)
  e.n_next = j->d_cnt + 4;
  e.n_rec = j->d_cnt + 5;
  e.n_stage = j->d_cnt + 6;
  es.n = j->d_cnt + 7;     // (d_cnt + 8: entries that died in the call)
  e.n_mids = j->d_cnt + 9;
  e.n_mrg = j->d_cnt + 10;
  const u64 ns = std::max(std::max(m, l), q + n);
  CU(ctx, j->srt.reserve(own, ns, ns, j->s));
  size_t b = 0;
  CU(ctx, cub::DeviceScan::ExclusiveScan(nullptr, b, o.cnt, j->d_off, PjSatAdd{}, (u64)0, (int)(m + 1), j->s));
  CU(ctx, j->srt.grow_cub(own, b + 256));
  CU(ctx, j->hm[0].reserve(own, m, m));
  CU(ctx, j->hm[1].reserve(own, m, m));
  CU(ctx, j->hl.reserve(own, l, l));
  CU(ctx, own.host(&j->h_mids, m));
  k_spjwin_init<<<ctx->sm_count * 4, 256, 0, j->s>>>(t);
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaStreamSynchronize(j->s));
  *out = jp.release();
  return BW_OK;
}

void bw_spjwin_destroy(bw_spjwin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  if (j->s) cudaStreamSynchronize(j->s);
  delete j;  // j->own releases every buffer and the stream
}

static JwParams spjwin_params(bw_spjwin* j, u64 epoch) {
  JwParams p{};
  p.emit_mode = j->spec.emit_mode;
  p.ordered = j->spec.ordered;
  p.wait = j->spec.wait_us;
  p.now = j->now;
  p.epoch = epoch;
  p.ord = j->calls++;
  p.batch_no = j->batch_no;
  return p;
}

#define SPJWIN_REFUSE_FAILED(j) \
  if ((j)->failed) CTX_FAIL((j)->ctx, BW_ERR_STATE, "session product join: an earlier call failed on the device; the join is unusable")

// K8's drain (failure, released handles, queue count), then the counts only this join keeps
static bw_status spjwin_drain(bw_spjwin* j) {
  const bool pending = j->undrained;
  bw_status st = jwin_drain(j);
  if (st != BW_OK || !pending) return st;
  j->n_meta = j->h_cnt[1];
  j->n_rec = j->h_cnt[5];
  j->n_stage = j->h_cnt[6];
  j->n_store = j->h_cnt[7];
  j->dead += j->h_cnt[8];
  j->n_mrg = j->h_cnt[10];
  CU(j->ctx, cudaMemsetAsync(j->d_cnt + 8, 0, 8, j->s));
  return BW_OK;
}

// Before a call that can play `rows` values (and ordered the queued entries): room in the release buffer, and in the
// store for one entry per value (K9's compaction and growth).  Called after the drain: nothing on the stream reads them.
static bw_status spjwin_room(bw_spjwin* j, u64 rows) {
  bw_status st = jwin_room(j, rows);
  if (st != BW_OK) return st;
  return store_room(j, rows + (j->spec.ordered ? j->nq : 0));
}

// The emit buffers the per-key kernels see.  One entry may be staged once per hop of a merge chain, so no bound on a
// call's staging is known before it runs: the kernels' stage records only reserve their ranges (no limit checked here),
// and spjwin_gather grows the buffer to what they reserved before anything is written there.
static SpEmit spjwin_walk_emit(const bw_spjwin* j) {
  SpEmit e = j->e;
  e.max_stage = ~0ULL;
  return e;
}

// after the per-key kernels of a call: room in staging for their stage records (what earlier calls staged is kept), then
// stage, retag and kill along every hop, and release (k_spjwin_gather)
static bw_status spjwin_gather(bw_spjwin* j, const JwParams& p) {
  bw_ctx* ctx = j->ctx;
  SpEmit& e = j->e;
  CU(ctx, cudaMemcpyAsync(j->h_cnt + 13, e.n_stage, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaMemcpyAsync(j->h_err + 2, j->t.err, 4, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 need = j->h_cnt[13];
  if (!j->h_err[2] && need > e.max_stage) {  // (after a failed call the gather does nothing and the drain reports it)
    const u64 grow = std::max<u64>(need, 2 * e.max_stage);
    e.max_stage = 0;
    CU(ctx, collect_grow_keep(j, &e.stage, j->n_stage, grow));
    e.max_stage = grow;
  }
  k_spjwin_gather<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, j->es, p, j->n_rec, j->n_meta, j->n_mrg, j->d_cnt + 8);
  CU(ctx, cudaGetLastError());
  return BW_OK;
}

// ordered mode: sort the pool's due entries into play order (K8's sort); then flush every woken key (k_spjwin_flush)
static bw_status spjwin_flush(bw_spjwin* j, const JwParams& p, u64 n) {
  bw_ctx* ctx = j->ctx;
  bw_status st = j->spec.ordered ? jwin_sort_pool(j, j->t.j, p, n) : BW_OK;
  if (st != BW_OK) return st;
  SpEmit e = spjwin_walk_emit(j);
  e.next = j->pool2;
  k_spjwin_flush<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, e, j->es, p, j->pool, j->srt.perm);
  CU(ctx, cudaGetLastError());
  if (j->spec.ordered) std::swap(j->pool, j->pool2);  // the next call reads what this flush carried over (count: jwin_drain)
  return spjwin_gather(j, p);
}

bw_status bw_spjwin_apply_device(bw_spjwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles,
                                 const int64_t* d_ts_us, uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (!j) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SPJWIN_REFUSE_FAILED(j);
  if (rows > j->spec.max_batch_rows) CTX_FAIL(ctx, BW_ERR_SPEC, "session product join: rows > max_batch_rows");
  if (rows && (!d_keys || !d_side || !d_handles || !d_ts_us)) CTX_FAIL(ctx, BW_ERR_SPEC, "session product join: NULL column");
  if (j->batch_no && epoch < j->last_epoch) CTX_FAIL(ctx, BW_ERR_STATE, "session product join: epochs must not decrease");
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = spjwin_drain(j);
  if (st != BW_OK) return st;
  j->last_epoch = epoch;
  if (system_now_us > j->now) j->now = system_now_us;  // `now_getter()` never goes backwards (windowing.py:250-261)
  const JwParams p = spjwin_params(j, epoch);
  j->batch_no++;
  if (rows == 0) return BW_OK;
  if ((st = spjwin_room(j, rows)) != BW_OK) return st;
  j->outstanding += rows;
  st = keyed_group(ctx, j->k, d_keys, rows, j->s);
  if (st != BW_OK) return st;
  k_spjwin_apply<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t, spjwin_walk_emit(j), j->es, p, j->pool, j->nq, j->k.d_ksorted, j->k.d_isorted,
                                                      j->k.d_head, d_handles, d_side, d_ts_us, j->d_late, rows);
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  if (j->spec.ordered) return spjwin_flush(j, p, j->nq + rows);
  return spjwin_gather(j, p);
}

static bw_status spjwin_apply_device_fn(bw_spjwin* j, const uint64_t* d_keys, const uint8_t* d_side, const uint64_t* d_handles,
                                        const int64_t* d_ts_us, uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  bw_status st = bw_spjwin_apply_device(j, d_keys, d_side, d_handles, d_ts_us, rows, epoch, system_now_us);
  if (st != BW_OK) return st;
  return spjwin_drain(j);  // (jwin_apply_host drains once more: then nothing is pending)
}

bw_status bw_spjwin_apply(bw_spjwin* j, const uint64_t* keys, const uint8_t* side, const uint64_t* handles, const int64_t* ts_us,
                          uint64_t rows, uint64_t epoch, int64_t system_now_us) {
  if (j) {
    SPJWIN_REFUSE_FAILED(j);
    bw_status st = spjwin_drain(j);  // (before jwin_apply_host's own drain, which would skip this join's counts)
    if (st != BW_OK) return st;
  }
  return jwin_apply_host(j, keys, side, handles, ts_us, rows, epoch, system_now_us, spjwin_apply_device_fn);
}

// advance / eof: the events in the reference's order (order_perm), K14's row counts and saturating scan; the host grows
// the output to the total; K14's k_pjwin_expand writes every row in that order
static bw_status spjwin_expand(bw_spjwin* j, u64 nd, u64* total) {
  bw_ctx* ctx = j->ctx;
  *total = 0;
  if (!nd) return BW_OK;
  SortScratch& x = j->srt;
  bw_status st = order_perm(ctx, x, j->s, nd, j->e.key, j->e.seq, j->e.ord, nullptr, std::max<u64>(j->calls - j->first_call, 1), j->first_call,
                            nullptr);
  if (st != BW_OK) return st;
  const int grid = ctx->sm_count * 4;
  const PjOrdered o = j->o;
  k_pjwin_count<<<grid, 256, 0, j->s>>>(j->e, o, j->spec.sides, x.perm, nd);
  CU(ctx, cudaMemsetAsync(o.cnt + nd, 0, 8, j->s));
  size_t tb = x.cub_bytes;
  CU(ctx, cub::DeviceScan::ExclusiveScan(x.cub, tb, o.cnt, j->d_off, PjSatAdd{}, (u64)0, (int)(nd + 1), j->s));
  CU(ctx, cudaMemcpyAsync(j->h_cnt + 12, j->d_off + nd, 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 n = j->h_cnt[12];
  if (n > j->spec.max_product_rows) {
    j->failed = true;
    CTX_FAIL(ctx, BW_ERR_CAPACITY, "session product join ran out of capacity: %llu product rows since the last advance, more than "
             "max_product_rows (%llu)", (unsigned long long)n, (unsigned long long)j->spec.max_product_rows);
  }
  if (n > j->rows_cap) {
    j->rows_cap = 0;
    for (u64** c : {&j->rows.key, &j->rows.wid, &j->rows.h0, &j->rows.h1, &j->rows.h2, &j->rows.h3, &j->rows.mask, &j->rows.epoch})
      CU(ctx, j->own.regrow(Owner::DEV, c, n));
    j->rows_cap = n;
  }
  CU(ctx, j->hd[0].reserve(j->own, n, n));
  CU(ctx, j->hd[1].reserve(j->own, n, n));
  k_pjwin_expand<<<ctx->sm_count * 8, 256, 0, j->s>>>(o, j->d_off, nd, j->spec.sides, j->e.stage, j->rows, n);
  const u64* src[] = {j->rows.key, j->rows.wid, j->rows.h0, j->rows.h1, j->rows.h2, j->rows.h3, j->rows.mask, j->rows.epoch};
  for (int c = 0; c < 8; ++c) CU(ctx, cudaMemcpyAsync(j->hd[c / 5].col[c % 5], src[c], n * 8, cudaMemcpyDeviceToHost, j->s));
  *total = n;
  return BW_OK;
}

static bw_status spjwin_collect(bw_spjwin* j, bw_sjwin_rows* out) {
  bw_ctx* ctx = j->ctx;
  bw_status st = spjwin_drain(j);
  if (st != BW_OK) return st;
  CU(ctx, cudaMemcpyAsync(j->h_cnt, j->d_cnt, 88, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  const u64 nd = j->h_cnt[0], nm = j->h_cnt[1], nl = j->h_cnt[2], nmid = j->h_cnt[9];  // all within bounds: the drain passed
  u64 n = 0;
  if ((st = spjwin_expand(j, nd, &n)) != BW_OK) return st;
  const SpEmit& e = j->e;
  const u64* meta[] = {e.m_key, e.m_wid, (const u64*)e.m_open, (const u64*)e.m_close, e.m_epoch, e.m_mcnt, e.m_moff};
  const u64* late[] = {e.l_key, e.l_wid, e.l_epoch, e.l_act, e.l_row};
  if ((st = jwin_ship(j, nm, e.m_key, e.m_seq, e.m_ord, meta, 7, j->hm)) != BW_OK) return st;
  if ((st = jwin_ship(j, nl, e.l_key, e.l_seq, e.l_ord, late, 5, &j->hl)) != BW_OK) return st;
  if (nmid) CU(ctx, cudaMemcpyAsync(j->h_mids, e.mids, nmid * 8, cudaMemcpyDeviceToHost, j->s));
  CU(ctx, cudaGetLastError());
  CU(ctx, cudaMemsetAsync(j->d_cnt, 0, 24, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 5, 0, 16, j->s));
  CU(ctx, cudaMemsetAsync(j->d_cnt + 9, 0, 8, j->s));
  CU(ctx, cudaStreamSynchronize(j->s));
  j->n_rec = j->n_meta = j->n_stage = 0;
  // merged ids in meta row order
  j->merged_off.assign(nm + 1, 0);
  j->merged_ids.resize(nmid);
  const u64 *cnt = j->hm[1].col[0], *off = j->hm[1].col[1];
  for (u64 r = 0; r < nm; ++r) {
    j->merged_off[r + 1] = j->merged_off[r] + cnt[r];
    std::copy(j->h_mids + off[r], j->h_mids + off[r] + cnt[r], j->merged_ids.begin() + j->merged_off[r]);
  }
  j->first_call = j->calls;
  out->n_down = n;
  out->down_key = j->hd[0].col[0];
  out->down_window_id = (const int64_t*)j->hd[0].col[1];
  out->down_handle[0] = j->hd[0].col[2];
  out->down_handle[1] = j->hd[0].col[3];
  out->down_handle[2] = j->hd[0].col[4];
  out->down_handle[3] = j->hd[1].col[0];
  out->down_mask = j->hd[1].col[1];
  out->down_epoch = j->hd[1].col[2];
  out->n_meta = nm;
  out->meta_key = j->hm[0].col[0];
  out->meta_window_id = (const int64_t*)j->hm[0].col[1];
  out->meta_open_us = (const int64_t*)j->hm[0].col[2];
  out->meta_close_us = (const int64_t*)j->hm[0].col[3];
  out->meta_epoch = j->hm[0].col[4];
  out->merged_off = j->merged_off.data();
  out->merged_ids = j->merged_ids.data();
  out->n_late = nl;
  out->late_key = j->hl.col[0];
  out->late_epoch = j->hl.col[2];
  out->late_activation = j->hl.col[3];
  out->late_row = j->hl.col[4];
  // handed out until the next advance / eof, then cleared
  j->released.swap(j->released_out);
  j->released.clear();
  out->n_released = j->released_out.size();
  out->released = j->released_out.data();
  return BW_OK;
}

// notify phase or EOF: wake the keys (K8's k_jwin_mark with the session notify_at), then flush them (ordered: through
// the pool)
static bw_status spjwin_wake(bw_spjwin* j, int eof) {
  bw_ctx* ctx = j->ctx;
  bw_status st = spjwin_drain(j);
  if (st != BW_OK) return st;
  if ((st = spjwin_room(j, 0)) != BW_OK) return st;
  const JwParams p = spjwin_params(j, j->last_epoch);
  k_jwin_mark<<<ctx->sm_count * 8, 256, 0, j->s>>>(j->t.j, (const SpRec*)j->t.rec, p, eof, SjNotifyAt{j->t.gap});
  CU(ctx, cudaGetLastError());
  j->undrained = true;
  return spjwin_flush(j, p, j->nq);
}

bw_status bw_spjwin_advance(bw_spjwin* j, int64_t system_now_us, bw_sjwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SPJWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  if (system_now_us > 0) {
    if (system_now_us > j->now) j->now = system_now_us;
    bw_status st = spjwin_wake(j, 0);
    if (st != BW_OK) return st;
  }
  return spjwin_collect(j, out);
}

bw_status bw_spjwin_eof(bw_spjwin* j, bw_sjwin_rows* out) {
  if (!j || !out) return BW_ERR_SPEC;
  bw_ctx* ctx = j->ctx;
  SPJWIN_REFUSE_FAILED(j);
  CU(ctx, cudaSetDevice(ctx->device));
  bw_status st = spjwin_wake(j, 1);
  if (st != BW_OK) return st;
  return spjwin_collect(j, out);
}
