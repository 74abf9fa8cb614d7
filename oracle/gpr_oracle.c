/*
 * gpr_oracle.c — CPU restatement of gpu-pruner's idle decision.  TEST INFRASTRUCTURE ONLY
 * (see gpr_oracle.h: parity unpinned; nothing in the product path may use this file).
 *
 * What is restated, line by line (reference paths relative to the reference repository):
 *
 *   gpu-pruner/src/query.promql.j2:16-20  max_over_time(DCGM_FI_DEV_GPU_UTIL{pod != ""}[Nm]) / 100
 *   gpu-pruner/src/query.promql.j2:9,21   sum by (Hostname, container, pod, namespace, gpu, modelName)
 *                                         -> one series per (pod, gpu) cell: identity
 *   gpu-pruner/src/query.promql.j2:35     == 0   (filter; -0.0 passes, NaN fails)
 *   gpu-pruner/src/query.promql.j2:36-44  unless on (pod, namespace) (max_over_time(POWER[Nm]) >= T)
 *   gpu-pruner/src/main.rs:416-437        HashSet<(pod, namespace)> dedup = ANY-GPU fold
 *   gpu-pruner/src/main.rs:473-510        Pending / no timestamp / created >= now - lookback => skip
 *
 * max_over_time follows Prometheus promql/functions.go funcMaxOverTime (external to the
 * reference tree, restated from its published algorithm): start from the first sample,
 * replace when `cur > max || isnan(max)`; a series with no sample in the window yields no
 * output element.  All arithmetic in float64, as in Prometheus; the f32 matrix is widened
 * per element.  Plain scalar C, no intrinsics: this is also "the reference CPU loop" timed
 * as the baseline.
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE /* sched_getaffinity / pthread_setaffinity_np for the timed baseline's pool */
#endif
#include "gpr_oracle.h"

#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

/* --------------------------------------------------------------------------------------
 * max_over_time  (query.promql.j2:16,20,39; Prometheus funcMaxOverTime)
 * ------------------------------------------------------------------------------------ */
double gpo_max_over_time(const float *row, uint32_t n) {
  uint32_t i = 0;
  /* samples that are "not there" are not part of the range vector */
  while (i < n && isnan(row[i])) ++i;
  if (i == n) return NAN; /* no sample in the window: series absent from the result */
  double m = (double)row[i];
  for (++i; i < n; ++i) {
    double v = (double)row[i];
    if (isnan(v)) continue; /* missing step */
    if (v > m || isnan(m)) m = v;
  }
  return m;
}

static int power_clause_enabled(const float *power, double thr) {
  /* Jinja `{%- if args.power_threshold %}` (query.promql.j2:36): None and 0.0 are falsy */
  return power != NULL && thr != 0.0 && !isnan(thr);
}

static void decide_range(const float *util, const float *power, const uint8_t *eligible,
                         const int64_t *created, int64_t cutoff, uint32_t p0, uint32_t p1,
                         uint32_t G, uint32_t T, uint64_t ld, double thr, uint32_t *dbits,
                         uint32_t *cbits, float *smax, uint64_t counts[3]) {
  const int use_power = power_clause_enabled(power, thr);
  uint64_t n_series = 0, n_cand = 0, n_dec = 0;
  for (uint32_t p = p0; p < p1; ++p) {
    uint32_t idle_series = 0;
    int veto = 0;
    for (uint32_t g = 0; g < G; ++g) {
      const uint64_t r = (uint64_t)p * G + g;
      const double m = gpo_max_over_time(util + r * ld, T);
      if (smax) smax[r] = (float)m; /* exact: m is one of the f32 inputs (or NaN) */
      /* `== 0` filter, query.promql.j2:35.  (x / 100 == 0) <=> (x == 0) for every
       * non-denormal x, and DCGM_FI_DEV_GPU_UTIL is an integer percentage.           */
      if (m == 0.0) ++idle_series;
      if (use_power) {
        const double w = gpo_max_over_time(power + r * ld, T);
        if (w >= thr) veto = 1; /* NaN >= thr is false: absent power series never vetoes */
      }
    }
    /* unless on (pod, namespace): pod-wide veto; dedup: pod is a candidate if >= 1 series
     * survived (main.rs:430-435)                                                       */
    const int candidate = idle_series > 0 && !veto;
    int elig = 1;
    if (eligible && !eligible[p]) elig = 0;            /* Pending / missing ts, main.rs:473-492 */
    if (created && created[p] >= cutoff) elig = 0;     /* main.rs:508-510 */
    const int decision = candidate && elig;
    if (candidate) {
      n_series += idle_series;
      ++n_cand;
      if (cbits) cbits[p >> 5] |= 1u << (p & 31);
    }
    if (decision) {
      ++n_dec;
      if (dbits) dbits[p >> 5] |= 1u << (p & 31);
    }
  }
  counts[0] = n_series;
  counts[1] = n_cand;
  counts[2] = n_dec;
}

static void zero_bits(uint32_t *b, uint32_t P) {
  if (b) memset(b, 0, (size_t)((P + 31) / 32) * sizeof(uint32_t));
}

int gpo_decide(const float *util, const float *power, const uint8_t *eligible,
               const int64_t *created, int64_t cutoff, uint32_t P, uint32_t G, uint32_t T,
               uint64_t ld, double thr, uint32_t *dbits, uint32_t *cbits, float *smax,
               uint64_t counts[3]) {
  uint64_t c[3];
  if (!util && P * G > 0) return -1;
  if (ld == 0) ld = T;
  zero_bits(dbits, P);
  zero_bits(cbits, P);
  decide_range(util, power, eligible, created, cutoff, 0, P, G, T, ld, thr, dbits, cbits, smax, c);
  if (counts) memcpy(counts, c, sizeof c);
  return 0;
}

/* ------------------------------ threaded wrapper ------------------------------------- */
typedef struct {
  const float *util, *power;
  const uint8_t *eligible;
  const int64_t *created;
  int64_t cutoff;
  uint32_t p0, p1, G, T;
  uint64_t ld;
  double thr;
  uint32_t *dbits, *cbits, *vbits;
  float *smax;
  uint64_t counts[3];
  /* synthetic streaming mode */
  int synth, use_power, use_elig;
  uint64_t seed, pod_offset;
  void *aux; /* other job kinds run through the same pool (gpo_synth_fill) */
} job_t;

static void *decide_job(void *arg) {
  job_t *j = (job_t *)arg;
  decide_range(j->util, j->power, j->eligible, j->created, j->cutoff, j->p0, j->p1, j->G, j->T,
               j->ld, j->thr, j->dbits, j->cbits, j->smax, j->counts);
  return NULL;
}

/* split [0,P) into n contiguous ranges whose boundaries are multiples of 32 pods, so no two
 * threads ever touch the same bitmap word                                                  */
static uint32_t split32(uint32_t P, int n, int i) {
  const uint64_t words = ((uint64_t)P + 31) / 32;
  uint64_t w = words * (uint64_t)i / (uint64_t)n;
  uint64_t p = w * 32;
  return (uint32_t)(p > P ? P : p);
}

/* Persistent worker pool: the timed CPU baseline must not pay 128 pthread_create calls per pass.
 * Worker i (1..n-1) runs job i of the current batch; the caller runs job 0. */
static struct {
  pthread_mutex_t mu;
  pthread_cond_t cv_start, cv_done;
  pthread_t *th;
  int *ids;
  int n;               /* workers alive (excluding the caller) */
  unsigned long gen;   /* batch generation */
  int n_jobs, pending;
  void *(*fn)(void *);
  job_t *jobs;
} g_pool = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER,
            NULL, NULL, 0, 0, 0, 0, NULL, NULL};

/* Optional pinning for the timed baseline (gpo_pool_pin): worker i stays on the i-th CPU this
 * process may run on, so the pages a worker first touches in gpo_synth_fill are the ones the same
 * worker streams in gpo_decide_mt (same pod split), whatever the box's NUMA layout. */
static volatile int g_pin = 0;

static void pin_self(int id) {
  cpu_set_t allowed, one;
  if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return;
  const int n = CPU_COUNT(&allowed);
  if (n <= 0) return;
  int want = id % n, seen = 0;
  for (int c = 0; c < CPU_SETSIZE; ++c) {
    if (!CPU_ISSET(c, &allowed)) continue;
    if (seen++ == want) {
      CPU_ZERO(&one);
      CPU_SET(c, &one);
      pthread_setaffinity_np(pthread_self(), sizeof one, &one);
      return;
    }
  }
}

void gpo_pool_pin(int on) { g_pin = on ? 1 : 0; }

static void *pool_worker(void *arg) {
  const int id = *(int *)arg; /* 1-based */
  unsigned long seen = 0;
  int pinned = 0;
  pthread_mutex_lock(&g_pool.mu);
  for (;;) {
    while (g_pool.gen == seen) pthread_cond_wait(&g_pool.cv_start, &g_pool.mu);
    seen = g_pool.gen;
    if (g_pin && !pinned) pin_self(id), pinned = 1;
    if (id < g_pool.n_jobs) {
      job_t *job = &g_pool.jobs[id];
      void *(*fn)(void *) = g_pool.fn;
      pthread_mutex_unlock(&g_pool.mu);
      fn(job);
      pthread_mutex_lock(&g_pool.mu);
      if (--g_pool.pending == 0) pthread_cond_signal(&g_pool.cv_done);
    }
  }
  return NULL;
}

static int pool_grow(int want_workers) {
  if (want_workers <= g_pool.n) return 0;
  pthread_t *th = (pthread_t *)realloc(g_pool.th, sizeof(pthread_t) * (size_t)want_workers);
  int *ids = (int *)malloc(sizeof(int) * (size_t)want_workers); /* stable storage per growth step */
  if (!th || !ids) return -1;
  g_pool.th = th;
  for (int i = g_pool.n; i < want_workers; ++i) {
    ids[i] = i + 1;
    if (pthread_create(&g_pool.th[i], NULL, pool_worker, &ids[i]) != 0) return -1;
    pthread_detach(g_pool.th[i]);
    g_pool.n = i + 1;
  }
  g_pool.ids = ids;
  return 0;
}

static int run_jobs(job_t *jobs, int n, void *(*fn)(void *)) {
  if (n <= 1) {
    fn(&jobs[0]);
    return 0;
  }
  pthread_mutex_lock(&g_pool.mu);
  if (pool_grow(n - 1) != 0) {
    pthread_mutex_unlock(&g_pool.mu);
    return -1;
  }
  g_pool.jobs = jobs, g_pool.fn = fn, g_pool.n_jobs = n, g_pool.pending = n - 1;
  ++g_pool.gen;
  pthread_cond_broadcast(&g_pool.cv_start);
  pthread_mutex_unlock(&g_pool.mu);
  fn(&jobs[0]);
  pthread_mutex_lock(&g_pool.mu);
  while (g_pool.pending > 0) pthread_cond_wait(&g_pool.cv_done, &g_pool.mu);
  pthread_mutex_unlock(&g_pool.mu);
  return 0;
}

int gpo_decide_mt(int n_threads, const float *util, const float *power, const uint8_t *eligible,
                  const int64_t *created, int64_t cutoff, uint32_t P, uint32_t G, uint32_t T,
                  uint64_t ld, double thr, uint32_t *dbits, uint32_t *cbits, float *smax,
                  uint64_t counts[3]) {
  if (n_threads < 1) n_threads = 1;
  if (ld == 0) ld = T;
  zero_bits(dbits, P);
  zero_bits(cbits, P);
  job_t *jobs = (job_t *)calloc((size_t)n_threads, sizeof(job_t));
  if (!jobs) return -1;
  for (int i = 0; i < n_threads; ++i) {
    job_t *j = &jobs[i];
    j->util = util, j->power = power, j->eligible = eligible, j->created = created;
    j->cutoff = cutoff, j->G = G, j->T = T, j->ld = ld, j->thr = thr;
    j->dbits = dbits, j->cbits = cbits, j->smax = smax;
    j->p0 = split32(P, n_threads, i);
    j->p1 = split32(P, n_threads, i + 1);
  }
  int rc = run_jobs(jobs, n_threads, decide_job);
  if (counts) {
    counts[0] = counts[1] = counts[2] = 0;
    for (int i = 0; i < n_threads; ++i)
      for (int k = 0; k < 3; ++k) counts[k] += jobs[i].counts[k];
  }
  free(jobs);
  return rc;
}

/* --------------------------------------------------------------------------------------
 * Synthetic DCGM universe.  Independent restatement of the recipe in DESIGN.md §synthetic
 * (SURVEY.md §8(d)): counter-based, every cell a pure function of (seed, series, t).
 * ------------------------------------------------------------------------------------ */
static uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

#define TAG_SERIES 0x5345524945530001ull
#define TAG_CELL 0x43454C4C00000002ull
#define TAG_POWER 0x504F574552000003ull
#define TAG_ELIG 0x454C494700000004ull

enum { CLS_IDLE = 0, CLS_BURST = 1, CLS_ACTIVE = 2, CLS_GAPPY = 3 };

typedef struct {
  int cls;
  uint32_t a;  /* burst index, or gappy prefix covers t <= a */
  uint64_t b;  /* burst value = 1 + b % 100; gappy tail is active iff b & 1 */
} series_t;

static series_t series_of(uint64_t seed, uint64_t s, uint32_t T) {
  const uint64_t hs = mix64(mix64(seed ^ TAG_SERIES) ^ s);
  const uint32_t c = (uint32_t)(hs % 100);
  series_t r;
  r.cls = c < 30 ? CLS_IDLE : c < 40 ? CLS_BURST : c < 95 ? CLS_ACTIVE : CLS_GAPPY;
  r.a = (uint32_t)((hs >> 8) % T);
  r.b = hs >> 40;
  return r;
}

static float util_cell(uint64_t kcell, const series_t *sr, uint64_t s, uint32_t t, uint32_t T) {
  const uint64_t hc = mix64(kcell ^ (s * (uint64_t)T + t));
  if (hc % 1000 == 0) return NAN; /* scrape gap, 0.1 % */
  const float v_active = ((hc >> 10) & 1) ? (float)(1 + ((hc >> 11) % 100)) : 0.0f;
  switch (sr->cls) {
    case CLS_IDLE: return 0.0f;
    case CLS_BURST: return t == sr->a ? (float)(1 + sr->b % 100) : 0.0f;
    case CLS_ACTIVE: return v_active;
    default: /* gappy / young pod: leading run of missing samples */
      if (t <= sr->a) return NAN;
      return (sr->b & 1) ? v_active : 0.0f;
  }
}

static float power_cell(uint64_t kpow, const series_t *sr, uint64_t s, uint32_t t, uint32_t T) {
  const uint64_t hp = mix64(kpow ^ (s * (uint64_t)T + t));
  if (hp % 1000 == 0) return NAN;
  const int low = sr->cls == CLS_IDLE || (sr->cls == CLS_GAPPY && !(sr->b & 1));
  return low ? (float)(40 + (hp >> 10) % 31) : (float)(70 + (hp >> 10) % 631);
}

float gpo_synth_cell(uint64_t seed, int plane, uint64_t s, uint32_t t, uint32_t T) {
  const series_t sr = series_of(seed, s, T);
  return plane == 0 ? util_cell(mix64(seed ^ TAG_CELL), &sr, s, t, T)
                    : power_cell(mix64(seed ^ TAG_POWER), &sr, s, t, T);
}

uint8_t gpo_synth_eligible_pod(uint64_t seed, uint64_t pod) {
  return (uint8_t)((mix64(mix64(seed ^ TAG_ELIG) ^ pod) % 100) >= 5);
}

static void fill_row(uint64_t seed, int plane, uint64_t s, uint32_t T, float *dst) {
  const series_t sr = series_of(seed, s, T);
  const uint64_t k = mix64(seed ^ (plane == 0 ? TAG_CELL : TAG_POWER));
  if (plane == 0)
    for (uint32_t t = 0; t < T; ++t) dst[t] = util_cell(k, &sr, s, t, T);
  else
    for (uint32_t t = 0; t < T; ++t) dst[t] = power_cell(k, &sr, s, t, T);
}

typedef struct {
  uint64_t seed, pod_offset, ld;
  int plane;
  float *dst;
  uint32_t p0, p1, G, T;
} fill_job_t;

static void *fill_job(void *arg) {
  fill_job_t *j = (fill_job_t *)((job_t *)arg)->aux;
  for (uint32_t p = j->p0; p < j->p1; ++p)
    for (uint32_t g = 0; g < j->G; ++g) {
      const uint64_t local = (uint64_t)p * j->G + g;
      const uint64_t s = (j->pod_offset + p) * j->G + g;
      fill_row(j->seed, j->plane, s, j->T, j->dst + local * j->ld);
    }
  return NULL;
}

int gpo_synth_fill(int n_threads, uint64_t seed, int plane, float *dst, uint64_t pod_offset,
                   uint32_t P, uint32_t G, uint32_t T, uint64_t ld) {
  if (n_threads < 1) n_threads = 1;
  if (ld == 0) ld = T;
  /* same pool and same pod split as gpo_decide_mt: with pinned workers every page is first touched by
   * the thread that later streams it */
  job_t *jobs = (job_t *)calloc((size_t)n_threads, sizeof(job_t));
  fill_job_t *fj = (fill_job_t *)calloc((size_t)n_threads, sizeof(fill_job_t));
  if (!jobs || !fj) {
    free(jobs), free(fj);
    return -1;
  }
  for (int i = 0; i < n_threads; ++i) {
    fill_job_t *j = &fj[i];
    j->seed = seed, j->pod_offset = pod_offset, j->ld = ld, j->plane = plane, j->dst = dst;
    j->G = G, j->T = T;
    j->p0 = split32(P, n_threads, i);
    j->p1 = split32(P, n_threads, i + 1);
    jobs[i].aux = j;
  }
  const int rc = run_jobs(jobs, n_threads, fill_job);
  free(jobs), free(fj);
  return rc;
}

int gpo_synth_eligible(uint64_t seed, uint8_t *dst, uint64_t pod_offset, uint32_t P) {
  for (uint32_t p = 0; p < P; ++p) dst[p] = gpo_synth_eligible_pod(seed, pod_offset + p);
  return 0;
}

/* streaming decision: regenerate each row, never materialise the tensor */
static void *synth_job(void *arg) {
  job_t *j = (job_t *)arg;
  const uint32_t T = j->T, G = j->G;
  float *urow = (float *)malloc(sizeof(float) * T);
  float *wrow = (float *)malloc(sizeof(float) * T);
  uint64_t n_series = 0, n_cand = 0, n_dec = 0;
  const int use_power = j->use_power && j->thr != 0.0 && !isnan(j->thr);
  for (uint32_t p = j->p0; p < j->p1 && urow && wrow; ++p) {
    uint32_t idle_series = 0;
    int veto = 0;
    for (uint32_t g = 0; g < G; ++g) {
      const uint64_t s = (j->pod_offset + p) * G + g;
      fill_row(j->seed, 0, s, T, urow);
      const double m = gpo_max_over_time(urow, T);
      if (j->smax) j->smax[(uint64_t)p * G + g] = (float)m;
      if (m == 0.0) ++idle_series;
      if (use_power) {
        fill_row(j->seed, 1, s, T, wrow);
        if (gpo_max_over_time(wrow, T) >= j->thr) veto = 1;
      }
    }
    if (veto && j->vbits) j->vbits[p >> 5] |= 1u << (p & 31);
    const int candidate = idle_series > 0 && !veto;
    const int elig = j->use_elig ? gpo_synth_eligible_pod(j->seed, j->pod_offset + p) : 1;
    if (candidate) {
      n_series += idle_series;
      ++n_cand;
      if (j->cbits) j->cbits[p >> 5] |= 1u << (p & 31);
    }
    if (candidate && elig) {
      ++n_dec;
      if (j->dbits) j->dbits[p >> 5] |= 1u << (p & 31);
    }
  }
  free(urow), free(wrow);
  j->counts[0] = n_series, j->counts[1] = n_cand, j->counts[2] = n_dec;
  return NULL;
}

int gpo_decide_synth(int n_threads, uint64_t seed, uint64_t pod_offset, uint32_t P, uint32_t G,
                     uint32_t T, int use_power, double thr, int use_elig, uint32_t *dbits,
                     uint32_t *cbits, uint64_t counts[3]) {
  return gpo_decide_synth_ex(n_threads, seed, pod_offset, P, G, T, use_power, thr, use_elig, dbits, cbits, NULL,
                             NULL, counts);
}

int gpo_decide_synth_ex(int n_threads, uint64_t seed, uint64_t pod_offset, uint32_t P, uint32_t G,
                        uint32_t T, int use_power, double thr, int use_elig, uint32_t *dbits,
                        uint32_t *cbits, float *smax, uint32_t *vbits, uint64_t counts[3]) {
  if (n_threads < 1) n_threads = 1;
  zero_bits(dbits, P);
  zero_bits(cbits, P);
  zero_bits(vbits, P);
  job_t *jobs = (job_t *)calloc((size_t)n_threads, sizeof(job_t));
  if (!jobs) return -1;
  for (int i = 0; i < n_threads; ++i) {
    job_t *j = &jobs[i];
    j->G = G, j->T = T, j->thr = thr, j->dbits = dbits, j->cbits = cbits, j->smax = smax, j->vbits = vbits;
    j->seed = seed, j->pod_offset = pod_offset, j->use_power = use_power, j->use_elig = use_elig;
    j->p0 = split32(P, n_threads, i);
    j->p1 = split32(P, n_threads, i + 1);
  }
  int rc = run_jobs(jobs, n_threads, synth_job);
  if (counts) {
    counts[0] = counts[1] = counts[2] = 0;
    for (int i = 0; i < n_threads; ++i)
      for (int k = 0; k < 3; ++k) counts[k] += jobs[i].counts[k];
  }
  free(jobs);
  return rc;
}

int gpo_hardware_threads(void) {
  cpu_set_t allowed; /* the CPUs this process may actually use (cgroup / taskset aware) */
  if (sched_getaffinity(0, sizeof allowed, &allowed) == 0 && CPU_COUNT(&allowed) > 0)
    return CPU_COUNT(&allowed);
  long n = sysconf(_SC_NPROCESSORS_ONLN);
  return n > 0 ? (int)n : 1;
}
