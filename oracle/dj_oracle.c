/*
 * dj_oracle.c -- CPU ORACLE for the distributed repartitioned inner-join hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (distributed-join_b200/csrc) never calls into this file and fails loudly without its
 * CUDA library.
 *
 * It restates, in plain C, the algorithm the reference executes on its hot path.  The
 * reference (rapidsai/distributed-join @ 26e84fee) delegates all device arithmetic to
 * cuDF 0.19 (not vendored: Dockerfile:18-19 `cudf=0.19`), so each function cites the
 * reference CALL SITE it follows plus the published algorithm it restates:
 *
 *   murmur3_x86_32 on the 8 key bytes  -- cudf::hash_id::HASH_MURMUR3,
 *        call sites src/distributed_join.cpp:211-225, src/shuffle_on.cpp:59-60
 *        (Austin Appleby's public-domain MurmurHash3_x86_32, len = 8).
 *   row hash = hash_combine(0, h)       -- cuDF 0.19 row_hasher, first column (SURVEY App. B).
 *   partition id = row_hash % nparts    -- cudf::hash_partition, same call sites.
 *   inner join (multimap, left++right)  -- cudf::inner_join, src/distributed_join.cpp:71-83,
 *        output schema asserted by test/compare_against_analytical.cu:44-54.
 *   batch/bucket -> rank mapping        -- src/distributed_join.cpp:247-266.
 *   known-selectivity generator         -- generate_dataset/generate_dataset.cuh:47-135,163-260
 *        and src/generate_table.cuh:155-272, restated with a counter-based RNG (Philox4x32-10)
 *        and a Feistel permutation so CPU and GPU produce bit-identical tables (the
 *        reference's cuRAND stream depends on the SM count and is not reproducible).
 *   analytical generator                -- test/compare_against_analytical.cu:64-81.
 *
 * PINNING.  Join results (cardinality, row multiset) are pinned by the reference's own
 * tests: G1 analytical cardinalities size/5 (test/compare_against_analytical.cu:152,194-201),
 * G3 equality with a single-node join (test/compare_against_single_gpu.cu:163-205), G5 the
 * generator's selectivity invariant.  The murmur3 step is pinned by known answers checked
 * bit-equal against sklearn.utils.murmurhash3_32 (tests/golden/murmur3_kat.json).
 * PARITY UNPINNED for the key -> partition-id assignment only: no reference test pins it
 * (test/test_shuffle_on.cpp:78-83 uses HASH_IDENTITY and checks congruence only) and cuDF
 * 0.19's row_hasher is not in the reference tree.  Join results are invariant to it.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <time.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------ hashing */

static inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

static inline uint32_t fmix32(uint32_t h)
{
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}

/* MurmurHash3_x86_32 of the 8 little-endian bytes of `key`. */
ORACLE_API uint32_t oracle_murmur3_i64(int64_t key, uint32_t seed)
{
  const uint32_t c1 = 0xcc9e2d51u, c2 = 0x1b873593u;
  uint64_t u  = (uint64_t)key;
  uint32_t h1 = seed;
  for (int i = 0; i < 2; i++) {
    uint32_t k1 = (uint32_t)(u >> (32 * i));
    k1 *= c1;
    k1 = rotl32(k1, 15);
    k1 *= c2;
    h1 ^= k1;
    h1 = rotl32(h1, 13);
    h1 = h1 * 5 + 0xe6546b64u;
  }
  h1 ^= 8u;
  return fmix32(h1);
}

/* hash ids mirror cudf::hash_id as used by the reference (src/shuffle_on.hpp:49,
 * test/test_shuffle_on.cpp uses HASH_IDENTITY). */
enum { ORACLE_HASH_IDENTITY = 0, ORACLE_HASH_MURMUR3 = 1 };

/* cuDF 0.19 row_hasher for a single key column: hash_combine(0, element_hash). */
ORACLE_API uint32_t oracle_row_hash_i64(int64_t key, uint32_t seed, int hash_id)
{
  uint32_t h = (hash_id == ORACLE_HASH_MURMUR3) ? oracle_murmur3_i64(key, seed) : (uint32_t)key;
  return h + 0x9e3779b9u;
}

ORACLE_API void oracle_partition_ids_i64(
  const int64_t* keys, int64_t n, uint32_t seed, int hash_id, int nparts, int32_t* out)
{
  for (int64_t i = 0; i < n; i++)
    out[i] = (int32_t)(oracle_row_hash_i64(keys[i], seed, hash_id) % (uint32_t)nparts);
}

/* cudf::hash_partition restated: stable counting sort of (key, payload) by partition id;
 * offsets has nparts+1 entries (the reference appends num_rows itself,
 * src/distributed_join.cpp:232-233). */
ORACLE_API void oracle_hash_partition_i64(const int64_t* keys,
                                          const int64_t* payload,
                                          int64_t n,
                                          uint32_t seed,
                                          int hash_id,
                                          int nparts,
                                          int64_t* out_keys,
                                          int64_t* out_payload,
                                          int64_t* offsets)
{
  int64_t* cursor = (int64_t*)calloc((size_t)nparts + 1, sizeof(int64_t));
  for (int64_t i = 0; i < n; i++)
    cursor[oracle_row_hash_i64(keys[i], seed, hash_id) % (uint32_t)nparts + 1]++;
  for (int p = 0; p < nparts; p++) cursor[p + 1] += cursor[p];
  memcpy(offsets, cursor, ((size_t)nparts + 1) * sizeof(int64_t));
  for (int64_t i = 0; i < n; i++) {
    uint32_t p       = oracle_row_hash_i64(keys[i], seed, hash_id) % (uint32_t)nparts;
    int64_t dst      = cursor[p]++;
    out_keys[dst]    = keys[i];
    out_payload[dst] = payload[i];
  }
  free(cursor);
}

/* ------------------------------------------------------------------ inner join */

static inline uint64_t mix64(uint64_t x)
{
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

static int64_t next_pow2(int64_t x)
{
  int64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

/* Chained hash table over build rows; returns heads/next (caller frees). */
typedef struct {
  int64_t* head;
  int64_t* next;
  int64_t mask;
} chain_table;

static chain_table chain_build(const int64_t* bk, int64_t nb)
{
  chain_table t;
  int64_t cap = next_pow2(nb * 2 + 16);
  t.mask      = cap - 1;
  t.head      = (int64_t*)malloc((size_t)cap * sizeof(int64_t));
  t.next      = (int64_t*)malloc((size_t)(nb > 0 ? nb : 1) * sizeof(int64_t));
  for (int64_t i = 0; i < cap; i++) t.head[i] = -1;
  for (int64_t i = 0; i < nb; i++) {
    int64_t s = (int64_t)(mix64((uint64_t)bk[i]) & (uint64_t)t.mask);
    t.next[i] = t.head[s];
    t.head[s] = i;
  }
  return t;
}

/*
 * Inner equi-join, multimap semantics, output columns left ++ right =
 * (left key, left payload, right key, right payload).  Either side empty -> 0 rows
 * (src/distributed_join.cpp:76-82).  Pass out_* = NULL to count only.  Returns the
 * cardinality; writes at most `capacity` rows.
 */
ORACLE_API int64_t oracle_inner_join_i64(const int64_t* lk,
                                         const int64_t* lp,
                                         int64_t nl,
                                         const int64_t* rk,
                                         const int64_t* rp,
                                         int64_t nr,
                                         int64_t* out_lk,
                                         int64_t* out_lp,
                                         int64_t* out_rk,
                                         int64_t* out_rp,
                                         int64_t capacity)
{
  if (nl == 0 || nr == 0) return 0;
  chain_table t = chain_build(lk, nl);
  int64_t n_out = 0;
  for (int64_t j = 0; j < nr; j++) {
    int64_t s = (int64_t)(mix64((uint64_t)rk[j]) & (uint64_t)t.mask);
    for (int64_t i = t.head[s]; i >= 0; i = t.next[i]) {
      if (lk[i] == rk[j]) {
        if (out_lk && n_out < capacity) {
          out_lk[n_out] = lk[i];
          out_lp[n_out] = lp[i];
          out_rk[n_out] = rk[j];
          out_rp[n_out] = rp[j];
        }
        n_out++;
      }
    }
  }
  free(t.head);
  free(t.next);
  return n_out;
}

/* Order-independent 128-bit checksum of a 4-column row multiset: (sum of h1(row), sum of
 * h2(row)) mod 2^64 with two independent row mixers.  Shared definition with the CUDA
 * library's dj_multiset_checksum so full-size results can be compared without sorting. */
static inline void row_digest(int64_t a, int64_t b, int64_t c, int64_t d, uint64_t* s1, uint64_t* s2)
{
  uint64_t x = mix64((uint64_t)a + 0x9e3779b97f4a7c15ULL);
  x          = mix64(x ^ (uint64_t)b);
  x          = mix64(x + (uint64_t)c);
  x          = mix64(x ^ (uint64_t)d);
  uint64_t y = mix64((uint64_t)d * 0xd6e8feb86659fd93ULL + 1);
  y          = mix64(y + (uint64_t)c);
  y          = mix64(y ^ (uint64_t)b);
  y          = mix64(y + (uint64_t)a);
  *s1 += x;
  *s2 += y;
}

ORACLE_API void oracle_multiset_checksum4(const int64_t* c0,
                                          const int64_t* c1,
                                          const int64_t* c2,
                                          const int64_t* c3,
                                          int64_t n,
                                          uint64_t* out2)
{
  uint64_t s1 = 0, s2 = 0;
#pragma omp parallel for reduction(+ : s1, s2) schedule(static)
  for (int64_t i = 0; i < n; i++) row_digest(c0[i], c1[i], c2[i], c3[i], &s1, &s2);
  out2[0] = s1;
  out2[1] = s2;
}

/* ------------------------------------------------------------------ generators */

/* Philox4x32-10 (Salmon et al., SC'11) -- counter-based, identical on CPU and GPU. */
static inline void philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4])
{
  uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3];
  uint32_t k0 = key[0], k1 = key[1];
  for (int r = 0; r < 10; r++) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

static inline double u01(uint32_t hi, uint32_t lo)
{
  return (double)((((uint64_t)hi << 32) | lo) >> 11) * (1.0 / 9007199254740992.0);
}

typedef struct {
  int64_t nb;        /* build rows per source rank                                        */
  int64_t np;        /* probe rows per source rank                                        */
  int64_t rand_max;  /* per-rank key range [0, rand_max] (benchmark/distributed_join.cu:187) */
  double selectivity;
  uint64_t seed;     /* reference cuRAND seed is 1234 (generate_dataset.cuh:44)           */
  int32_t unique;    /* unique build keys (generate_dataset.cuh:64-84) or not (:85-86)    */
  int32_t pad;
} oracle_gen_params;

enum { GEN_STREAM_BUILD = 0, GEN_STREAM_PROBE = 1 };

static inline void gen_draw(const oracle_gen_params* g, int stream, int attempt, int src_rank,
                            int64_t row, double* x0, double* x1)
{
  uint32_t ctr[4] = {(uint32_t)row, (uint32_t)((uint64_t)row >> 32),
                     (uint32_t)stream | ((uint32_t)attempt << 8), (uint32_t)src_rank};
  uint32_t key[2] = {(uint32_t)g->seed, (uint32_t)(g->seed >> 32)};
  uint32_t o[4];
  philox4x32_10(ctr, key, o);
  *x0 = u01(o[0], o[1]);
  *x1 = u01(o[2], o[3]);
}

/* Pseudo-random permutation of [0, L): balanced Feistel network on the next even number
 * of bits, cycle-walked into range.  perm(0..nb-1) is the unique build-key set in random
 * order (the reference's lottery, generate_dataset.cuh:64-84); perm(nb..L-1) is the
 * complement the miss keys are drawn from (:228-245). */
static inline uint64_t feistel_perm(uint64_t x, uint64_t L, uint64_t seed, uint32_t src_rank)
{
  int bits = 2;
  while (((uint64_t)1 << bits) < L) bits += 2;
  const int half      = bits / 2;
  const uint32_t mask = (uint32_t)(((uint64_t)1 << half) - 1);
  do {
    uint32_t l = (uint32_t)(x >> half) & mask, r = (uint32_t)x & mask;
    for (uint32_t rnd = 0; rnd < 6; rnd++) {
      uint32_t f = fmix32(r * 0x9E3779B1u + (uint32_t)seed + 0x7F4A7C15u * (rnd + 1) +
                          0x85EBCA77u * src_rank + (uint32_t)(seed >> 32));
      uint32_t t = l ^ (f & mask);
      l          = r;
      r          = t;
    }
    x = ((uint64_t)l << half) | r;
  } while (x >= L);
  return x;
}

static inline int64_t clampi(int64_t v, int64_t hi) { return v > hi ? hi : v; }

/* Build key of local row `row` on source rank `src` (before the rank key offset). */
static inline int64_t gen_build_local(const oracle_gen_params* g, int src, int64_t row)
{
  const int64_t L = g->rand_max + 1;
  if (g->unique) return (int64_t)feistel_perm((uint64_t)row, (uint64_t)L, g->seed, (uint32_t)src);
  double x0, x1;
  gen_draw(g, GEN_STREAM_BUILD, 0, src, row, &x0, &x1);
  return clampi((int64_t)(x0 * (double)g->rand_max), g->rand_max);
}

ORACLE_API void oracle_build_bitmap(const oracle_gen_params* g, int src, uint32_t* bitmap)
{
  const int64_t L = g->rand_max + 1;
  memset(bitmap, 0, (size_t)((L + 31) / 32) * sizeof(uint32_t));
  for (int64_t i = 0; i < g->nb; i++) {
    int64_t k = gen_build_local(g, src, i);
    bitmap[k >> 5] |= 1u << (k & 31);
  }
}

/* Probe key of local row `row` on source rank `src`; *hit tells whether it was a hit draw
 * (generate_dataset.cuh:110-132).  bitmap is only read when !unique. */
static inline int64_t gen_probe_local(const oracle_gen_params* g, int src, int64_t row,
                                      const uint32_t* bitmap, int* hit)
{
  const int64_t L = g->rand_max + 1;
  double x0, x1;
  gen_draw(g, GEN_STREAM_PROBE, 0, src, row, &x0, &x1);
  const int no_miss_keys = g->unique && (L - g->nb <= 0);
  if (x0 < g->selectivity || no_miss_keys) {
    *hit      = 1;
    int64_t j = clampi((int64_t)(x1 * (double)g->nb), g->nb - 1);
    return gen_build_local(g, src, j);
  }
  *hit = 0;
  if (g->unique) {
    int64_t m = clampi((int64_t)(x1 * (double)(L - g->nb)), L - g->nb - 1);
    return (int64_t)feistel_perm((uint64_t)(g->nb + m), (uint64_t)L, g->seed, (uint32_t)src);
  }
  /* duplicates allowed: rejection-sample a key absent from the build bitmap */
  int64_t c = clampi((int64_t)(x1 * (double)L), L - 1);
  for (int attempt = 1; attempt < 64 && (bitmap[c >> 5] >> (c & 31) & 1u); attempt++) {
    gen_draw(g, GEN_STREAM_PROBE, attempt, src, row, &x0, &x1);
    c = clampi((int64_t)(x1 * (double)L), L - 1);
  }
  for (int64_t step = 0; step < L && (bitmap[c >> 5] >> (c & 31) & 1u); step++) c = (c + 1) % L;
  return c;
}

/*
 * Generate rows [row_begin, row_begin+count) of source rank `src`'s local build (which=0)
 * or probe (which=1) table, with the distributed wrapper's offsets applied
 * (src/generate_table.cuh:192-202): key += rand_max*src, payload = row + n_rank*src.
 * Returns the number of hit draws among generated probe rows (0 for build).
 */
ORACLE_API int64_t oracle_generate_rows(const oracle_gen_params* g, int which, int src,
                                        int64_t row_begin, int64_t count,
                                        const uint32_t* bitmap, int64_t* keys, int64_t* payload)
{
  int64_t hits         = 0;
  const int64_t n_rank = which ? g->np : g->nb;
#pragma omp parallel for reduction(+ : hits) schedule(static)
  for (int64_t t = 0; t < count; t++) {
    int64_t row = row_begin + t;
    int64_t k;
    if (which == 0) {
      k = gen_build_local(g, src, row);
    } else {
      int hit = 0;
      k       = gen_probe_local(g, src, row, bitmap, &hit);
      hits += hit;
    }
    if (keys) keys[t] = k + g->rand_max * (int64_t)src;
    if (payload) payload[t] = row + n_rank * (int64_t)src;
  }
  return hits;
}

/* Analytical tables of test/compare_against_analytical.cu:64-81: key = mult*i, payload = i. */
ORACLE_API void oracle_generate_analytical(int64_t mult, int64_t row_begin, int64_t count,
                                           int64_t* keys, int64_t* payload)
{
  for (int64_t t = 0; t < count; t++) {
    keys[t]    = mult * (row_begin + t);
    payload[t] = row_begin + t;
  }
}

/* ------------------------------------------------------------------ CPU baseline */

static double now_s(void)
{
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/*
 * The whole hot path on host cores, as the CPU baseline bench.py times: murmur3 hash
 * partition of both tables into `nparts` cache-sized partitions (the reference's
 * cudf::hash_partition step), then an independent hash inner join per partition (the
 * reference's per-rank cudf::inner_join), OpenMP-parallel over rows / partitions.
 * Returns the join cardinality; *seconds gets the wall time of partition+join;
 * checksum2 (optional) gets the multiset checksum of the output rows.
 */
ORACLE_API int64_t oracle_partitioned_join_omp(const int64_t* bk, const int64_t* bp, int64_t nb,
                                               const int64_t* pk, const int64_t* pp, int64_t np,
                                               int nparts, uint32_t seed, double* seconds,
                                               uint64_t* checksum2, int* threads_used)
{
  int nthreads = 1;
#ifdef _OPENMP
  nthreads = omp_get_max_threads();
#endif
  if (threads_used) *threads_used = nthreads;
  int64_t* bko = (int64_t*)malloc((size_t)(nb + 1) * 8);
  int64_t* bpo = (int64_t*)malloc((size_t)(nb + 1) * 8);
  int64_t* pko = (int64_t*)malloc((size_t)(np + 1) * 8);
  int64_t* ppo = (int64_t*)malloc((size_t)(np + 1) * 8);
  int64_t* boff = (int64_t*)calloc((size_t)nparts + 1, 8);
  int64_t* poff = (int64_t*)calloc((size_t)nparts + 1, 8);
  double t0 = now_s();

  /* parallel stable partition: per-thread histograms -> prefix -> scatter */
  for (int tbl = 0; tbl < 2; tbl++) {
    const int64_t* k = tbl ? pk : bk;
    const int64_t* p = tbl ? pp : bp;
    int64_t n        = tbl ? np : nb;
    int64_t* ko      = tbl ? pko : bko;
    int64_t* po      = tbl ? ppo : bpo;
    int64_t* off     = tbl ? poff : boff;
    int64_t* hist    = (int64_t*)calloc((size_t)nthreads * (size_t)nparts, 8);
#pragma omp parallel num_threads(nthreads)
    {
      int t = 0;
#ifdef _OPENMP
      t = omp_get_thread_num();
#endif
      int64_t lo = n * t / nthreads, hi = n * (t + 1) / nthreads;
      int64_t* h = hist + (size_t)t * nparts;
      for (int64_t i = lo; i < hi; i++)
        h[oracle_row_hash_i64(k[i], seed, ORACLE_HASH_MURMUR3) % (uint32_t)nparts]++;
#pragma omp barrier
#pragma omp single
      {
        int64_t run = 0;
        for (int q = 0; q < nparts; q++) {
          off[q] = run;
          for (int tt = 0; tt < nthreads; tt++) {
            int64_t c                     = hist[(size_t)tt * nparts + q];
            hist[(size_t)tt * nparts + q] = run;
            run += c;
          }
        }
        off[nparts] = run;
      }
      for (int64_t i = lo; i < hi; i++) {
        uint32_t q  = oracle_row_hash_i64(k[i], seed, ORACLE_HASH_MURMUR3) % (uint32_t)nparts;
        int64_t dst = h[q]++;
        ko[dst]     = k[i];
        po[dst]     = p[i];
      }
    }
    free(hist);
  }

  int64_t total = 0;
  uint64_t s1 = 0, s2 = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : total, s1, s2) num_threads(nthreads)
  for (int q = 0; q < nparts; q++) {
    int64_t b0 = boff[q], b1 = boff[q + 1], p0 = poff[q], p1 = poff[q + 1];
    if (b1 == b0 || p1 == p0) continue;
    chain_table t = chain_build(bko + b0, b1 - b0);
    for (int64_t j = p0; j < p1; j++) {
      int64_t s = (int64_t)(mix64((uint64_t)pko[j]) & (uint64_t)t.mask);
      for (int64_t i = t.head[s]; i >= 0; i = t.next[i]) {
        if (bko[b0 + i] == pko[j]) {
          total++;
          if (checksum2) {
            uint64_t a = 0, b = 0;
            row_digest(bko[b0 + i], bpo[b0 + i], pko[j], ppo[j], &a, &b);
            s1 += a;
            s2 += b;
          }
        }
      }
    }
    free(t.head);
    free(t.next);
  }
  double t1 = now_s();
  if (seconds) *seconds = t1 - t0;
  if (checksum2) {
    checksum2[0] = s1;
    checksum2[1] = s2;
  }
  free(bko); free(bpo); free(pko); free(ppo); free(boff); free(poff);
  return total;
}

ORACLE_API void oracle_set_threads(int n)
{
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

ORACLE_API int oracle_num_threads(void)
{
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
