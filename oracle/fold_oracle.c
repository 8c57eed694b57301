/*
 * fold_oracle.c -- plain-C restatement of the reference's windowed-fold path.
 * TEST INFRASTRUCTURE ONLY: linked/loaded solely by tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs.  The product
 * (bytewax_b200/) never touches it.
 *
 * Parity status: pinned -- tests/test_oracle_c.py checks this file against the
 * golden vectors generated from the reference's own Python logic
 * (tests/golden/window_fold_cases.json, made by oracle/gen_golden.py) and
 * against oracle/pyoracle.py on seeded inputs.
 *
 * What it follows (paths relative to the bytewax v0.21.1 source tree):
 *   per-activation grouping + ascending key-string order  src/operators.rs:755-806
 *   on_eof for every live key                              src/operators.rs:862-894
 *   event clock / watermark                                pysrc/bytewax/operators/windowing.py:263-287
 *   intersects / open_for / close_for                      windowing.py:611-654
 *   on_batch / _flush_queue (ordered + unordered)          windowing.py:1095-1133
 *   discard of an empty logic                              windowing.py:1110-1113
 * Times are int64 microseconds; values are int64 or double.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define UTC_MIN_US (-62135596800000000LL)
#define UTC_MAX_US (253402300799999999LL)

enum { RED_COUNT = 0, RED_SUM = 1, RED_MIN = 2, RED_MAX = 3, RED_MEAN = 4 };

typedef union {
  int64_t i;
  double f;
  uint64_t bits;
} val_t;

typedef struct {
  int64_t wid;
  val_t acc;
  uint64_t cnt;
  int has;
} win_t;

typedef struct {
  val_t v;
  int64_t ts;
} qent_t;

typedef struct {
  uint64_t key;
  int live;              /* logic exists */
  int64_t wm_base;       /* watermark_base (UTC_MIN when fresh) */
  win_t* wins;           /* open windows, first-opened order */
  int nwins, capwins;
  qent_t* queue;         /* ordered mode: items not yet due */
  int nq, capq;
  /* per-activation event list */
  int64_t ev_head, ev_tail;
  char keystr[24];
} kstate_t;

typedef struct {
  uint64_t* key;
  int64_t* wid;
  uint64_t* acc;
  uint64_t* cnt;
  uint64_t* act;
  size_t n, cap;
} rows_t;

typedef struct oracle {
  int reduction, is_float, ordered;
  int64_t length, offset, align, wait;
  /* open addressing key -> state index */
  uint64_t* slots; /* index+1, 0 = empty */
  size_t nslots;
  kstate_t* st;
  size_t nst, capst;
  rows_t closed, late;
  uint64_t act;
  /* scratch */
  int64_t* next;
  size_t capnext;
  size_t* touched;
  size_t captouched;
} oracle;

static uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

static int64_t floordiv(int64_t a, int64_t b) {
  int64_t q = a / b, r = a % b;
  return (r != 0 && ((r < 0) != (b < 0))) ? q - 1 : q;
}

static void rows_push(rows_t* r, uint64_t key, int64_t wid, uint64_t acc, uint64_t cnt, uint64_t act) {
  if (r->n == r->cap) {
    r->cap = r->cap ? r->cap * 2 : 1024;
    r->key = realloc(r->key, r->cap * 8);
    r->wid = realloc(r->wid, r->cap * 8);
    r->acc = realloc(r->acc, r->cap * 8);
    r->cnt = realloc(r->cnt, r->cap * 8);
    r->act = realloc(r->act, r->cap * 8);
  }
  r->key[r->n] = key;
  r->wid[r->n] = wid;
  r->acc[r->n] = acc;
  r->cnt[r->n] = cnt;
  r->act[r->n] = act;
  r->n++;
}

oracle* orc_create(int reduction, int is_float, int64_t length, int64_t offset, int64_t align, int64_t wait, int ordered) {
  oracle* o = calloc(1, sizeof *o);
  o->reduction = reduction;
  o->is_float = is_float;
  o->ordered = ordered;
  o->length = length;
  o->offset = offset;
  o->align = align;
  o->wait = wait;
  o->nslots = 1024;
  o->slots = calloc(o->nslots, 8);
  return o;
}

void orc_destroy(oracle* o) {
  if (!o) return;
  for (size_t i = 0; i < o->nst; ++i) {
    free(o->st[i].wins);
    free(o->st[i].queue);
  }
  free(o->st);
  free(o->slots);
  free(o->closed.key); free(o->closed.wid); free(o->closed.acc); free(o->closed.cnt); free(o->closed.act);
  free(o->late.key); free(o->late.wid); free(o->late.acc); free(o->late.cnt); free(o->late.act);
  free(o->next);
  free(o->touched);
  free(o);
}

static void grow_slots(oracle* o) {
  size_t n2 = o->nslots * 2;
  uint64_t* s2 = calloc(n2, 8);
  for (size_t i = 0; i < o->nst; ++i) {
    size_t h = mix64(o->st[i].key) & (n2 - 1);
    while (s2[h]) h = (h + 1) & (n2 - 1);
    s2[h] = i + 1;
  }
  free(o->slots);
  o->slots = s2;
  o->nslots = n2;
}

static size_t find_key(oracle* o, uint64_t key) {
  if ((o->nst + 1) * 2 > o->nslots) grow_slots(o);
  size_t h = mix64(key) & (o->nslots - 1);
  while (o->slots[h]) {
    size_t i = o->slots[h] - 1;
    if (o->st[i].key == key) return i;
    h = (h + 1) & (o->nslots - 1);
  }
  if (o->nst == o->capst) {
    o->capst = o->capst ? o->capst * 2 : 1024;
    o->st = realloc(o->st, o->capst * sizeof(kstate_t));
  }
  kstate_t* k = &o->st[o->nst];
  memset(k, 0, sizeof *k);
  k->key = key;
  k->ev_head = k->ev_tail = -1;
  snprintf(k->keystr, sizeof k->keystr, "%llu", (unsigned long long)key);
  o->slots[h] = o->nst + 1;
  return o->nst++;
}

static void fold_into(oracle* o, win_t* w, val_t v) {
  switch (o->reduction) {
    case RED_COUNT: w->acc.i += 1; break; /* windowing.py:1686 */
    case RED_SUM:
      if (!w->has) w->acc = v; /* reduce_window seeds with the first value, windowing.py:2268-2274 */
      else if (o->is_float) w->acc.f += v.f;
      else w->acc.i += v.i;
      break;
    case RED_MIN:
      if (!w->has) w->acc = v;
      else if (o->is_float) { if (v.f < w->acc.f) w->acc = v; }
      else if (v.i < w->acc.i) w->acc = v;
      break;
    case RED_MAX:
      if (!w->has) w->acc = v;
      else if (o->is_float) { if (v.f > w->acc.f) w->acc = v; }
      else if (v.i > w->acc.i) w->acc = v;
      break;
    case RED_MEAN: w->acc.f += o->is_float ? v.f : (double)v.i; break;
  }
  w->has = 1;
  w->cnt++;
}

/* open_for + on_value for every intersecting window, windowing.py:1064-1077 */
static void insert_value(oracle* o, kstate_t* k, val_t v, int64_t ts) {
  int64_t since = ts - o->align;
  int64_t w0 = floordiv(since - o->length, o->offset) + 1, w1 = floordiv(since, o->offset);
  for (int64_t wid = w0; wid <= w1; ++wid) {
    int j;
    for (j = 0; j < k->nwins; ++j)
      if (k->wins[j].wid == wid) break;
    if (j == k->nwins) {
      if (k->nwins == k->capwins) {
        k->capwins = k->capwins ? k->capwins * 2 : 4;
        k->wins = realloc(k->wins, k->capwins * sizeof(win_t));
      }
      memset(&k->wins[j], 0, sizeof(win_t));
      k->wins[j].wid = wid;
      k->nwins++;
    }
    fold_into(o, &k->wins[j], v);
  }
}

static int cmp_q(const void* a, const void* b) {
  const qent_t *x = a, *y = b;
  return (x->ts > y->ts) - (x->ts < y->ts);
}

/* _flush_queue, windowing.py:1095-1108 */
static void flush(oracle* o, kstate_t* k, int64_t watermark) {
  if (o->ordered) {
    /* due = ts <= watermark, stable sort by ts */
    int nd = 0;
    qent_t* due = malloc((k->nq ? k->nq : 1) * sizeof(qent_t));
    int keep = 0;
    for (int i = 0; i < k->nq; ++i) {
      if (k->queue[i].ts <= watermark) due[nd++] = k->queue[i];
      else k->queue[keep++] = k->queue[i];
    }
    k->nq = keep;
    /* stable: merge sort via qsort on (ts, original index) -- indices are already ascending in due[] */
    /* make it stable by a simple insertion sort (due lists are short in tests) or mergesort */
    if (nd > 1) {
      /* stable merge sort */
      qent_t* tmp = malloc(nd * sizeof(qent_t));
      for (int width = 1; width < nd; width *= 2) {
        for (int lo = 0; lo < nd; lo += 2 * width) {
          int mid = lo + width < nd ? lo + width : nd, hi = lo + 2 * width < nd ? lo + 2 * width : nd;
          int a = lo, b = mid, t = lo;
          while (a < mid && b < hi) tmp[t++] = (cmp_q(&due[b], &due[a]) < 0) ? due[b++] : due[a++];
          while (a < mid) tmp[t++] = due[a++];
          while (b < hi) tmp[t++] = due[b++];
        }
        memcpy(due, tmp, nd * sizeof(qent_t));
      }
      free(tmp);
    }
    for (int i = 0; i < nd; ++i) insert_value(o, k, due[i].v, due[i].ts);
    free(due);
  } else {
    for (int i = 0; i < k->nq; ++i) insert_value(o, k, k->queue[i].v, k->queue[i].ts);
    k->nq = 0;
  }
  /* close_for in first-opened order, windowing.py:645-654 */
  int keep = 0;
  for (int j = 0; j < k->nwins; ++j) {
    int64_t close = o->align + o->offset * k->wins[j].wid + o->length;
    if (close <= watermark) {
      rows_push(&o->closed, k->key, k->wins[j].wid, k->wins[j].acc.bits, k->wins[j].cnt, o->act);
    } else {
      k->wins[keep++] = k->wins[j];
    }
  }
  k->nwins = keep;
}

static void qpush(kstate_t* k, val_t v, int64_t ts) {
  if (k->nq == k->capq) {
    k->capq = k->capq ? k->capq * 2 : 8;
    k->queue = realloc(k->queue, k->capq * sizeof(qent_t));
  }
  k->queue[k->nq].v = v;
  k->queue[k->nq].ts = ts;
  k->nq++;
}

static __thread oracle* g_sort_o;
static int cmp_touched(const void* a, const void* b) {
  return strcmp(g_sort_o->st[*(const size_t*)a].keystr, g_sort_o->st[*(const size_t*)b].keystr);
}

/*
 * One activation (src/operators.rs:755-806).  vals: int64 or double per is_float
 * (may be NULL for count).  Only rows with route(key) == part (of nparts) are
 * processed when nparts > 1 (key-sharded workers).
 */
void orc_on_batch(oracle* o, const uint64_t* keys, const int64_t* ts, const void* vals, size_t n, int part, int nparts) {
  if (n > o->capnext) {
    o->capnext = n;
    o->next = realloc(o->next, n * 8);
  }
  size_t ntouched = 0;
  for (size_t i = 0; i < n; ++i) {
    if (nparts > 1 && (int)(((mix64(keys[i]) >> 32) * (uint64_t)nparts) >> 32) != part) continue;
    size_t ki = find_key(o, keys[i]);
    kstate_t* k = &o->st[ki];
    o->next[i] = -1;
    if (k->ev_head < 0) {
      k->ev_head = k->ev_tail = (int64_t)i;
      if (ntouched == o->captouched) {
        o->captouched = o->captouched ? o->captouched * 2 : 1024;
        o->touched = realloc(o->touched, o->captouched * sizeof(size_t));
      }
      o->touched[ntouched++] = ki;
    } else {
      o->next[k->ev_tail] = (int64_t)i;
      k->ev_tail = (int64_t)i;
    }
  }
  g_sort_o = o;
  qsort(o->touched, ntouched, sizeof(size_t), cmp_touched); /* BTreeMap<String,_> order */
  for (size_t t = 0; t < ntouched; ++t) {
    kstate_t* k = &o->st[o->touched[t]];
    if (!k->live) { /* builder(None): fresh clock, windower, logic */
      k->live = 1;
      k->wm_base = UTC_MIN_US;
    }
    int64_t watermark = k->wm_base;
    for (int64_t i = k->ev_head; i >= 0; i = o->next[i]) {
      val_t v;
      v.bits = 0;
      if (vals) v.bits = ((const uint64_t*)vals)[i];
      /* clock.on_item, windowing.py:263-287 (frozen system clock) */
      watermark = k->wm_base;
      if (ts[i] >= UTC_MIN_US + o->wait) { /* else: OverflowError branch */
        int64_t cand = ts[i] - o->wait;
        if (cand > watermark) {
          k->wm_base = cand;
          watermark = cand;
        }
      }
      if (ts[i] < watermark) { /* late, windowing.py:1125-1127 */
        int64_t since = ts[i] - o->align;
        int64_t w0 = floordiv(since - o->length, o->offset) + 1, w1 = floordiv(since, o->offset);
        for (int64_t wid = w0; wid <= w1; ++wid) rows_push(&o->late, k->key, wid, v.bits, (uint64_t)ts[i], o->act);
      } else {
        qpush(k, v, ts[i]);
      }
    }
    flush(o, k, watermark);
    k->ev_head = k->ev_tail = -1;
    if (k->nwins == 0 && k->nq == 0) k->live = 0; /* discard, windowing.py:1110-1113 */
  }
  o->act++;
}

void orc_on_eof(oracle* o) {
  size_t nl = 0;
  size_t* live = malloc((o->nst ? o->nst : 1) * sizeof(size_t));
  for (size_t i = 0; i < o->nst; ++i)
    if (o->st[i].live) live[nl++] = i;
  g_sort_o = o;
  qsort(live, nl, sizeof(size_t), cmp_touched);
  for (size_t t = 0; t < nl; ++t) {
    kstate_t* k = &o->st[live[t]];
    flush(o, k, UTC_MAX_US); /* windowing.py:1144-1151 */
    k->live = 0;
  }
  free(live);
  o->act++;
}

size_t orc_n_closed(const oracle* o) { return o->closed.n; }
size_t orc_n_late(const oracle* o) { return o->late.n; }
/* col: 0 key, 1 wid, 2 acc bits, 3 count (late: ts), 4 activation index */
const void* orc_closed_col(const oracle* o, int col) {
  switch (col) { case 0: return o->closed.key; case 1: return o->closed.wid; case 2: return o->closed.acc; case 3: return o->closed.cnt; default: return o->closed.act; }
}
const void* orc_late_col(const oracle* o, int col) {
  switch (col) { case 0: return o->late.key; case 1: return o->late.wid; case 2: return o->late.acc; case 3: return o->late.cnt; default: return o->late.act; }
}
void orc_clear_rows(oracle* o) { o->closed.n = 0; o->late.n = 0; }

/* ---- CPU baseline: config C1 (SURVEY.md 8d), key-sharded worker threads ---- */
static uint64_t splitmix64(uint64_t x) { return mix64(x + 0x9E3779B97F4A7C15ULL); }

void orc_gen_c1(uint64_t* keys, int64_t* ts, uint64_t* vals, uint64_t start, size_t n, uint64_t n_keys, int64_t align) {
  for (size_t i = 0; i < n; ++i) {
    uint64_t g = start + i;
    keys[i] = splitmix64(0x5EEDULL ^ g) % n_keys;
    vals[i] = g;
    ts[i] = align + (int64_t)g;
  }
}

typedef struct {
  oracle* o;
  const uint64_t* keys;
  const int64_t* ts;
  size_t n;
  int part, nparts;
} job_t;

static void* worker(void* p) {
  job_t* j = p;
  orc_on_batch(j->o, j->keys, j->ts, NULL, j->n, j->part, j->nparts);
  return NULL;
}

/* One activation on `nthreads` key-sharded oracles (the reference's worker model,
 * src/timely.rs:540-551: all items of a key reach the same worker). */
void orc_on_batch_mt(oracle** os, int nthreads, const uint64_t* keys, const int64_t* ts, size_t n) {
  pthread_t th[64];
  job_t jobs[64];
  if (nthreads > 64) nthreads = 64;
  for (int t = 0; t < nthreads; ++t) {
    jobs[t] = (job_t){os[t], keys, ts, n, t, nthreads};
    pthread_create(&th[t], NULL, worker, &jobs[t]);
  }
  for (int t = 0; t < nthreads; ++t) pthread_join(th[t], NULL);
}
