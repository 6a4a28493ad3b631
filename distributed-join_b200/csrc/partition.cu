// partition.cu -- radix / hash partition passes for sm_90a (H100).
//
// One "pass" splits every parent bucket (a contiguous row range of SoA int64 columns) into
// F child buckets, in three stream-ordered launches and no host synchronisation:
//
//   plan_kernel    tile tables: which (parent, chunk) every tile index maps to
//   hist_kernel    reads keys only (8 B/row): exact child-bucket sizes -> exclusive scan
//   scatter_kernel reads every column once, writes it once (algorithmic 16 B * (1+npay)/2
//                  per row in each direction): each CTA stages a tile of rows in shared
//                  memory sorted by child bucket, reserves the tile's slice of every child
//                  bucket with one global atomicAdd per non-empty bucket, and streams the
//                  sorted tile out so that a warp's stores land in contiguous runs.
//
// It replaces cudf::hash_partition (reference call sites src/distributed_join.cpp:213-225,
// src/shuffle_on.cpp:59-60) in mode 0, and is the join's private sub-partitioner in mode 1.
//
// The join's radix levels (mode 1, row output) run as BOUNDED passes instead (run_bounded_pass):
// no histogram.  bucket_bases_kernel gives every child bucket a capacity from its parent's row
// count (mean + z*sigma + margin: the bucket bits come from a strong mixing hash) and lays the
// buckets out with gaps; the scatter drops any run that would pass its bucket's capacity and flags
// the parent.  Its cursor atomics still count every row, so repair_bases_kernel turns a flagged
// parent's cursors into exact offsets inside the parent's region, and a second scatter re-runs over
// that parent's input segments only.  The repair kernels are always enqueued and return at once
// when no parent is flagged: no host synchronisation.
//
// Two scatter families:
//   * SoA -> SoA (scatter_tma_kernel / scatter_kernel): the public cudf::hash_partition
//     replacement, columns in, columns out.
//   * -> rows (scatter_rows_kernel): everything internal to the join.  Output is 16-byte
//     (key, payload) rows; each (tile, bucket) run leaves shared memory as ONE cp.async.bulk
//     shared->global copy, so the write-out costs no LDS/STG wavefronts at all and overlaps the
//     ranking of the next tile.  Input is either the caller's SoA columns or rows.
#include <cub/device/device_scan.cuh>

#include <cmath>
#include <cstdlib>

#include "dj_device.cuh"
#include "dj_internal.h"

namespace dj {

namespace {

constexpr int kHistThreads    = 512;
constexpr int kHistTileRows   = 32768;
constexpr int kScatterThreads = 512;
constexpr int kRowsPerThread  = 8;
constexpr int kScatterTile    = kScatterThreads * kRowsPerThread;  // 4096 rows


template <int MODE>
__device__ __forceinline__ int bucket_of(int64_t key, const PassDev& d)
{
  if (MODE == 0) {
    uint32_t h = row_hash_i64(key, d.seed, d.hash_id);
    return d.pow2 ? (int)(h & (uint32_t)(d.F - 1)) : (int)(h % (uint32_t)d.F);
  } else if (MODE == 1) {
    return (int)((local_hash_i64(key) >> d.shift) & (uint32_t)(d.F - 1));
  } else {
    // fused rank partition + first local radix level: destination-major bucket index
    const uint32_t h    = row_hash_i64(key, d.seed, d.hash_id);
    const uint32_t dest = d.pow2 ? (h & (uint32_t)(d.nparts - 1)) : (h % (uint32_t)d.nparts);
    return (int)((dest << d.sub_bits) | (local_hash_i64(key) >> (32 - d.sub_bits)));
  }
}

// largest p in [0, P) with prefix[p] <= t
__device__ __forceinline__ int find_parent(const int* prefix, int P, int t)
{
  int lo = 0, hi = P;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (prefix[mid] <= t) lo = mid; else hi = mid;
  }
  return lo;
}

// ---------------------------------------------------------------- plan
// One CTA: input segments -> tile prefix tables for the two tile sizes.  Segments come either
// explicitly (begin/end/parent arrays: e.g. the per-source pieces of a received table), from
// parent ranges (segment i = parent i), or are the single range [0, nrows).  With `keep`, a
// segment whose parent p has keep[p] == 0 is emptied (a bounded pass's repair re-plans its own
// segments in place this way: only overflowed parents keep their rows).
__global__ void plan_kernel(const int64_t* parent_begin_in, const int64_t* parent_end_in,
                            const int64_t* seg_begin_in, const int64_t* seg_end_in, const int* seg_parent_in,
                            int64_t nrows, int S, int scatter_tile, int64_t* seg_begin, int64_t* seg_end,
                            int* seg_parent, int* hist_tiles, int* scat_tiles, const int* keep)
{
  __shared__ int warp_sums[33];
  const int tid = threadIdx.x;
  int64_t lo = 0, hi = 0;
  if (tid < S) {
    int parent = tid;
    if (seg_begin_in) {
      lo     = seg_begin_in[tid];
      hi     = seg_end_in[tid];
      parent = seg_parent_in ? seg_parent_in[tid] : 0;
    } else if (parent_begin_in) {
      lo = parent_begin_in[tid];
      hi = parent_end_in[tid];
    } else {
      lo     = 0;
      hi     = nrows;
      parent = 0;
    }
    if (keep && !keep[parent]) hi = lo;
    seg_begin[tid]  = lo;
    seg_end[tid]    = hi;
    seg_parent[tid] = parent;
  }
  int64_t n = hi - lo;
  int ht    = (int)((n + kHistTileRows - 1) / kHistTileRows);
  int st    = (int)((n + scatter_tile - 1) / scatter_tile);
  int he = block_exclusive_scan<1024>(ht, warp_sums);
  if (tid < S) hist_tiles[tid] = he;
  if (tid == 0) hist_tiles[S] = warp_sums[32];
  __syncthreads();
  int se = block_exclusive_scan<1024>(st, warp_sums);
  if (tid < S) scat_tiles[tid] = se;
  if (tid == 0) scat_tiles[S] = warp_sums[32];
}

// Bucket offsets for a pass whose output is handed to NCCL: buckets are laid out in groups of
// `group` consecutive buckets (one group per destination rank); every group starts on a multiple
// of `align` rows, buckets inside a group are contiguous.  Single CTA, nb <= 1024.
__global__ void aligned_offsets_kernel(const unsigned long long* counts, int nb, int group, int align,
                                       int64_t* off, int64_t* cnt_out)
{
  __shared__ int warp_sums[33];
  __shared__ int s_excl[1025];   // exclusive scan of raw counts, in rows
  __shared__ int s_gstart[1025];  // padded start of every group, in units of `align` rows
  const int tid = threadIdx.x;
  const int c   = tid < nb ? (int)counts[tid] : 0;
  const int e   = block_exclusive_scan<1024>(c, warp_sums);
  if (tid < nb) s_excl[tid] = e;
  if (tid == 0) s_excl[nb] = warp_sums[32];
  __syncthreads();
  const int ngroups = nb / group;
  int padded        = 0;
  if (tid < ngroups) padded = (s_excl[(tid + 1) * group] - s_excl[tid * group] + align - 1) / align;
  const int ge = block_exclusive_scan<1024>(padded, warp_sums);
  if (tid < ngroups) s_gstart[tid] = ge;
  if (tid == 0) s_gstart[ngroups] = warp_sums[32];
  __syncthreads();
  if (tid < nb) {
    const int g = tid / group;
    off[tid]    = (int64_t)s_gstart[g] * align + (s_excl[tid] - s_excl[g * group]);
    if (cnt_out) cnt_out[tid] = c;
  }
  if (tid == 0) off[nb] = (int64_t)s_gstart[ngroups] * align;
}

// ---------------------------------------------------------------- histogram
template <int MODE, bool IN_ROWS>
__global__ void __launch_bounds__(kHistThreads) hist_kernel(PassDev d)
{
  extern __shared__ int s_hist[];
  __shared__ int s_parent;
  const int tid   = threadIdx.x;
  const int total = d.hist_tiles[d.S];
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    for (int i = tid; i < d.F; i += kHistThreads) s_hist[i] = 0;
    if (tid == 0) s_parent = find_parent(d.hist_tiles, d.S, t);
    __syncthreads();
    const int sg      = s_parent;
    const int p       = d.seg_parent[sg];
    const int64_t beg = d.seg_begin[sg] + (int64_t)(t - d.hist_tiles[sg]) * kHistTileRows;
    int64_t end       = beg + kHistTileRows;
    if (end > d.seg_end[sg]) end = d.seg_end[sg];
#pragma unroll 8
    for (int64_t i = beg + tid; i < end; i += kHistThreads)
      atomicAdd(&s_hist[bucket_of<MODE>(IN_ROWS ? d.in_rows[i].key : d.in_key[i], d)], 1);
    __syncthreads();
    for (int i = tid; i < d.F; i += kHistThreads) {
      int c = s_hist[i];
      if (c) atomicAdd(&d.counts[(size_t)p * d.F + i], (unsigned long long)c);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- scatter
// Dynamic shared memory layout (T = kScatterTile):
//   int4 srow[T] (key, payload 0) | int64 spay[NPAY-1][T] | int64 s_delta[F] | int s_start[F] |
//   uint16 sbkt[T]
// The sorted tile is kept as 16-byte rows so that the scattered write and the streaming read are
// single 128-bit shared-memory accesses (half the wavefronts of two 64-bit ones).
constexpr int kMaxBinsPerThread = (kMaxFanout + kScatterThreads - 1) / kScatterThreads;

__device__ __forceinline__ void prefetch_l2(const void* p)
{
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

template <int MODE, int NPAY, bool WARP_AGG>
__global__ void __launch_bounds__(kScatterThreads, 2) scatter_kernel(PassDev d)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int T  = kScatterTile;
  int4* srow       = reinterpret_cast<int4*>(smem_raw);
  int64_t* spay    = reinterpret_cast<int64_t*>(srow + T);
  int64_t* s_delta = spay + (size_t)(NPAY - 1) * T;
  int* s_start     = reinterpret_cast<int*>(s_delta + d.F);
  uint16_t* sbkt   = reinterpret_cast<uint16_t*>(s_start + d.F);
  __shared__ int warp_sums[33];
  __shared__ int s_parent, s_parent_next;

  const int tid   = threadIdx.x;
  const int lane  = tid & 31;
  const int F     = d.F;
  const int total = d.scat_tiles[d.S];
  const int bpt   = (F + kScatterThreads - 1) / kScatterThreads;

  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int tn = t + gridDim.x;  // this CTA's next tile: pulled into L2 while this one runs
    for (int i = tid; i < F; i += kScatterThreads) s_start[i] = 0;
    if (tid == 0) s_parent = find_parent(d.scat_tiles, d.S, t);
    if (tid == 32 && tn < total) s_parent_next = find_parent(d.scat_tiles, d.S, tn);
    __syncthreads();
    const int sg      = s_parent;
    const int p       = d.seg_parent[sg];
    const int64_t beg = d.seg_begin[sg] + (int64_t)(t - d.scat_tiles[sg]) * T;
    int64_t end       = beg + T;
    if (end > d.seg_end[sg]) end = d.seg_end[sg];
    const int tile_n = (int)(end - beg);

    if (tn < total) {
      const int pn       = s_parent_next;
      const int64_t nbeg = d.seg_begin[pn] + (int64_t)(tn - d.scat_tiles[pn]) * T;
      int64_t nend       = nbeg + T;
      if (nend > d.seg_end[pn]) nend = d.seg_end[pn];
      // T rows = T/16 lines of 128 B per column; one line per thread and column
      constexpr int kLines = T / 16;
      for (int l = tid; l < kLines; l += kScatterThreads) {
        const int64_t row = nbeg + (int64_t)l * 16;
        if (row < nend) {
          prefetch_l2(d.in_key + row);
#pragma unroll
          for (int c = 0; c < NPAY; c++) prefetch_l2(d.in_pay[c] + row);
        }
      }
    }

    // phase 1: load keys, bucket, rank inside the tile's bucket
    int64_t key[kRowsPerThread];
    uint32_t brank[kRowsPerThread];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; j++) {
      const int r = j * kScatterThreads + tid;
      key[j]      = r < tile_n ? d.in_key[beg + r] : 0;
    }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; j++) {
      const int r      = j * kScatterThreads + tid;
      const bool valid = r < tile_n;
      const int b      = valid ? bucket_of<MODE>(key[j], d) : 0;
      int rank;
      if (WARP_AGG) {
        // few buckets: one shared-memory atomic per (warp, bucket) instead of per row
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        rank                 = 0;
        if (valid) {
          const unsigned peers = __match_any_sync(vmask, b);
          const int leader     = __ffs(peers) - 1;
          int base             = 0;
          if (lane == leader) base = atomicAdd(&s_start[b], __popc(peers));
          base = __shfl_sync(peers, base, leader);
          rank = base + __popc(peers & lanemask_lt());
        }
      } else {
        rank = valid ? atomicAdd(&s_start[b], 1) : 0;
      }
      brank[j] = ((uint32_t)b << 16) | (uint32_t)rank;
    }
    __syncthreads();

    // phase 2: exclusive scan of the tile histogram; reserve the tile's slice of each bucket.
    // The global atomicAdd results are only consumed after phase 3, hiding their round trip.
    unsigned long long gres[kMaxBinsPerThread];
    int grun[kMaxBinsPerThread];
    {
      const int b0 = tid * bpt;
      int sum      = 0;
      for (int k = 0; k < bpt; k++)
        if (b0 + k < F) sum += s_start[b0 + k];
      int run = block_exclusive_scan<kScatterThreads>(sum, warp_sums);
#pragma unroll
      for (int k = 0; k < kMaxBinsPerThread; k++) {
        grun[k] = -1;
        if (k < bpt && b0 + k < F) {
          const int c     = s_start[b0 + k];
          s_start[b0 + k] = run;
          if (c) {
            gres[k] = atomicAdd(&d.cursor[(size_t)p * F + b0 + k], (unsigned long long)c);
            grun[k] = run;
          }
          run += c;
        }
      }
    }
    __syncthreads();

    // phase 3: rows into bucket-sorted order in shared memory (payloads straight from L2/HBM)
#pragma unroll
    for (int j = 0; j < kRowsPerThread; j++) {
      const int r = j * kScatterThreads + tid;
      if (r < tile_n) {
        const int b       = brank[j] >> 16;
        const int pos     = s_start[b] + (int)(brank[j] & 0xffffu);
        const int64_t pay = d.in_pay[0][beg + r];
        srow[pos]         = make_int4((int)(uint32_t)(uint64_t)key[j], (int)((uint64_t)key[j] >> 32),
                                      (int)(uint32_t)(uint64_t)pay, (int)((uint64_t)pay >> 32));
        sbkt[pos]         = (uint16_t)b;
#pragma unroll
        for (int c = 1; c < NPAY; c++) spay[(size_t)(c - 1) * T + pos] = d.in_pay[c][beg + r];
      }
    }
#pragma unroll
    for (int k = 0; k < kMaxBinsPerThread; k++)
      if (grun[k] >= 0) s_delta[tid * bpt + k] = (int64_t)gres[k] - grun[k];
    __syncthreads();

    // phase 4: stream the sorted tile out; consecutive threads hit consecutive addresses
    for (int i = tid; i < tile_n; i += kScatterThreads) {
      const int64_t dst = s_delta[sbkt[i]] + i;
      const int4 row    = srow[i];
      d.out_key[dst]    = (int64_t)(((uint64_t)(uint32_t)row.y << 32) | (uint32_t)row.x);
      d.out_pay[0][dst] = (int64_t)(((uint64_t)(uint32_t)row.w << 32) | (uint32_t)row.z);
#pragma unroll
      for (int c = 1; c < NPAY; c++) d.out_pay[c][dst] = spay[(size_t)(c - 1) * T + i];
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- scatter, TMA-staged
// One persistent 1024-thread CTA per SM for the key + one payload case.  Input tiles are
// pulled HBM -> shared memory by TMA bulk copies (cp.async.bulk + mbarrier) two tiles ahead,
// so the ranking / sorting phases never wait on global loads and HBM stays busy while they
// run; everything else follows scatter_kernel.  Destination rows are tracked as 32-bit
// offsets (tables < 2^32 rows).
struct TileDesc {
  int64_t beg;
  int n;
  int parent;
};

// Stages rows [beg, beg+n) of an 8-byte column: the TMA source must be 16-byte aligned, so the copy
// covers the aligned window around the rows (row `beg` lands at smem_dst[skip_of(col + beg)]).
// The window never leaves the column: when the column's last row sits in the low half of a
// 16-byte word, that row is copied by hand instead.  Two calls per tile and column:
//   issue == false  returns the bytes the TMA will deliver and performs the hand copy -- a plain
//                   shared-memory store by the issuing thread, BEFORE its mbarrier arrive
//                   (release), so consumers that pass the barrier see it;
//   issue == true   issues the TMA copy.
__device__ __forceinline__ uint32_t stage_column(int64_t* smem_dst, const int64_t* col, int64_t beg, int n,
                                                 int64_t col_rows, unsigned long long* bar, bool issue)
{
  const uintptr_t a   = reinterpret_cast<uintptr_t>(col + beg);
  const uintptr_t lo  = a & ~(uintptr_t)15;
  uintptr_t hi        = (a + (uintptr_t)n * 8 + 15) & ~(uintptr_t)15;
  const uintptr_t end = reinterpret_cast<uintptr_t>(col + col_rows);
  if (hi > end) {
    hi -= 16;
    if (!issue) smem_dst[(hi - lo) >> 3] = col[beg + n - 1];
  }
  const uint32_t bytes = (uint32_t)(hi - lo);
  if (issue && bytes) tma_load(smem_dst, reinterpret_cast<const void*>(lo), bytes, bar);
  return bytes;
}

// THREADS x RPT rows per tile, two TMA stages.
template <int THREADS, int RPT>
struct __align__(128) ScatterTmaSmem {
  static constexpr int T = THREADS * RPT;
  int64_t kst[2][T + 2];
  int64_t pst[2][T + 2];
  int4 srow[T];
  uint16_t sbkt[T];
  int s_start[kMaxFanout];
  uint32_t s_delta[kMaxFanout];
  unsigned long long full[2];
  TileDesc desc[2];
  int warp_sums[33];
};

template <int MODE, bool WARP_AGG, int THREADS, int RPT>
__global__ void __launch_bounds__(THREADS, 1) scatter_tma_kernel(PassDev d)
{
  using Smem = ScatterTmaSmem<THREADS, RPT>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& s           = *reinterpret_cast<Smem*>(smem_raw);
  constexpr int T   = THREADS * RPT;
  constexpr int BPT = (kMaxFanout + THREADS - 1) / THREADS;  // histogram bins per thread
  const int tid     = threadIdx.x;
  const int lane    = tid & 31;
  const int F       = d.F;
  const int total   = d.scat_tiles[d.S];

  // thread 0 walks this CTA's tiles two ahead of the consumers; segments only move forward
  int prod_parent = 0;
  auto issue_tile = [&](int k) {  // thread 0 only
    const int t = blockIdx.x + k * gridDim.x;
    if (t >= total) return;
    while (d.scat_tiles[prod_parent + 1] <= t) prod_parent++;
    const int64_t beg = d.seg_begin[prod_parent] + (int64_t)(t - d.scat_tiles[prod_parent]) * T;
    int64_t end       = beg + T;
    if (end > d.seg_end[prod_parent]) end = d.seg_end[prod_parent];
    const int st = k & 1, n = (int)(end - beg);
    s.desc[st]   = TileDesc{beg, n, d.seg_parent[prod_parent]};
    const uint32_t bytes = stage_column(s.kst[st], d.in_key, beg, n, d.in_total, &s.full[st], false) +
                           stage_column(s.pst[st], d.in_pay[0], beg, n, d.in_total, &s.full[st], false);
    mbar_expect_tx(&s.full[st], bytes);
    stage_column(s.kst[st], d.in_key, beg, n, d.in_total, &s.full[st], true);
    stage_column(s.pst[st], d.in_pay[0], beg, n, d.in_total, &s.full[st], true);
  };

  if (tid == 0) {
    mbar_init(&s.full[0], 1);
    mbar_init(&s.full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    issue_tile(0);
    issue_tile(1);
  }

  for (int k = 0; blockIdx.x + k * (int)gridDim.x < total; k++) {
    const int st = k & 1;
#pragma unroll
    for (int q = 0; q < BPT; q++)
      if (tid + q * THREADS < F) s.s_start[tid + q * THREADS] = 0;
    __syncthreads();  // previous tile fully written out; descriptors of this tile visible
    mbar_wait(&s.full[st], (k >> 1) & 1);
    const TileDesc td  = s.desc[st];
    const int tile_n   = td.n;
    const int64_t* kst = s.kst[st] + skip_of(d.in_key + td.beg);
    const int64_t* pst = s.pst[st] + skip_of(d.in_pay[0] + td.beg);

    // phase 1: keys from the staged tile -> bucket, rank inside the tile's bucket
    int64_t key[RPT];
    uint32_t brank[RPT];
#pragma unroll
    for (int j = 0; j < RPT; j++) {
      const int r = j * THREADS + tid;
      key[j]      = r < tile_n ? kst[r] : 0;
    }
#pragma unroll
    for (int j = 0; j < RPT; j++) {
      const int r      = j * THREADS + tid;
      const bool valid = r < tile_n;
      const int b      = valid ? bucket_of<MODE>(key[j], d) : 0;
      int rank;
      if (WARP_AGG) {
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        rank                 = 0;
        if (valid) {
          const unsigned peers = __match_any_sync(vmask, b);
          const int leader     = __ffs(peers) - 1;
          int base             = 0;
          if (lane == leader) base = atomicAdd(&s.s_start[b], __popc(peers));
          base = __shfl_sync(peers, base, leader);
          rank = base + __popc(peers & lanemask_lt());
        }
      } else {
        rank = valid ? atomicAdd(&s.s_start[b], 1) : 0;
      }
      brank[j] = ((uint32_t)b << 16) | (uint32_t)rank;
    }
    __syncthreads();

    // phase 2: exclusive scan of the tile histogram (BPT consecutive bins per thread); reserve
    // the tile's slice of every bucket -- the atomicAdd results are consumed after phase 3
    int cnt[BPT], run[BPT];
    unsigned long long gres[BPT];
    {
      int sum = 0;
#pragma unroll
      for (int q = 0; q < BPT; q++) {
        const int bin = tid * BPT + q;
        cnt[q]        = bin < F ? s.s_start[bin] : 0;
        sum += cnt[q];
      }
      int excl = block_exclusive_scan<THREADS>(sum, s.warp_sums);
#pragma unroll
      for (int q = 0; q < BPT; q++) {
        const int bin = tid * BPT + q;
        run[q]        = excl;
        gres[q]       = 0;
        if (bin < F) {
          s.s_start[bin] = excl;
          if (cnt[q]) gres[q] = atomicAdd(&d.cursor[(size_t)td.parent * F + bin], (unsigned long long)cnt[q]);
        }
        excl += cnt[q];
      }
    }
    __syncthreads();

    // phase 3: rows into bucket-sorted order (16-byte rows) in shared memory
#pragma unroll
    for (int j = 0; j < RPT; j++) {
      const int r = j * THREADS + tid;
      if (r < tile_n) {
        const int b       = brank[j] >> 16;
        const int pos     = s.s_start[b] + (int)(brank[j] & 0xffffu);
        const int64_t pay = pst[r];
        s.srow[pos] = make_int4((int)(uint32_t)(uint64_t)key[j], (int)((uint64_t)key[j] >> 32),
                                (int)(uint32_t)(uint64_t)pay, (int)((uint64_t)pay >> 32));
        s.sbkt[pos] = (uint16_t)b;
      }
    }
#pragma unroll
    for (int q = 0; q < BPT; q++)
      if (cnt[q]) s.s_delta[tid * BPT + q] = (uint32_t)gres[q] - (uint32_t)run[q];
    __syncthreads();  // sorted tile complete; the input stage is free again

    if (tid == 0) issue_tile(k + 2);

    // phase 4: stream the sorted tile out; consecutive threads hit consecutive addresses
#pragma unroll
    for (int j = 0; j < RPT; j++) {
      const int i = j * THREADS + tid;
      if (i < tile_n) {
        int4 row;
        asm volatile("ld.shared.v4.s32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(row.x), "=r"(row.y), "=r"(row.z), "=r"(row.w)
                     : "r"(smem_u32(&s.srow[i])));
        const int64_t k64  = (int64_t)(((uint64_t)(uint32_t)row.y << 32) | (uint32_t)row.x);
        const uint32_t dst = s.s_delta[s.sbkt[i]] + (uint32_t)i;
        d.out_key[dst]     = k64;
        d.out_pay[0][dst]  = (int64_t)(((uint64_t)(uint32_t)row.w << 32) | (uint32_t)row.z);
      }
    }
  }
}

// ---------------------------------------------------------------- scatter -> rows
// The join's internal partitioner: key + payload in (SoA columns or 16-byte rows), 16-byte rows
// out.  One persistent 1024-thread CTA per SM; per 4096-row tile:
//   TMA      the tile arrives in shared memory two tiles ahead (cp.async.bulk + mbarrier);
//   rank     every row: bucket = hash bits, rank = shared-memory atomicAdd on the bucket's counter
//            (experiments/mb_smem_rank.cu compares it with warp-aggregated ranking);
//   reserve  one thread per bucket: global atomicAdd reserves the run's slice of the bucket (the
//            result is not needed until the copy-out), block scan of the counters;
//   sort     every row is written to its bucket-sorted position as one STS.128;
//   copy-out the thread owning bucket b issues ONE cp.async.bulk shared->global for the run
//            (16-byte aligned on both sides because rows are 16 bytes): the TMA engine streams the
//            tile out while the CTA already ranks the next tile.  No LDS/STG for the write-out.
// Three CTA barriers per tile (four in the LEAN == false variant).  The sorted tile is single-buffered: cp.async.bulk.wait_group.read
// (shared-memory side of the copies done) is awaited just before the next tile's sort.
template <int THREADS, int RPT, bool IN_ROWS>
struct __align__(128) ScatterRowsSmem {
  static constexpr int T = THREADS * RPT;
  // input stages: IN_ROWS: Row[2][T]; else int64 key[2][T+2] + pay[2][T+2] (aligned windows)
  unsigned char in[IN_ROWS ? 2 * T * 16 : 4 * (T + 2) * 8];
  Row srow[T];
  int s_cnt[2][kMaxFanout];
  int s_start[kMaxFanout];
  unsigned long long full[2];
  TileDesc desc[2];
  int warp_sums[32];
};

// LEAN (default): three CTA barriers per tile instead of four -- bucket starts are assembled from the
// in-warp prefix (shared memory) plus the prefix over warp totals, which every warp keeps in
// registers (lane l holds the prefix of warp l) and reads with a shuffle -- and the tile producer is
// lane 0 of the LAST warp, which owns the fewest buckets, so its dependent descriptor loads are off
// the other warps' critical path.  LEAN == false is the first version of the kernel, kept selectable
// (DJ_SCATTER_LEAN=0).
template <int MODE, bool IN_ROWS, int THREADS, int RPT, bool LEAN>
__global__ void __launch_bounds__(THREADS, 1) scatter_rows_kernel(PassDev d)
{
  static_assert(THREADS >= kMaxFanout, "one thread owns one bucket");
  static_assert(!LEAN || THREADS == 1024, "LEAN keeps one warp-total prefix per lane: exactly 32 warps");
  constexpr int kProducer = LEAN ? THREADS - 32 : 0;
  using Smem = ScatterRowsSmem<THREADS, RPT, IN_ROWS>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& s         = *reinterpret_cast<Smem*>(smem_raw);
  constexpr int T = THREADS * RPT;
  const int tid   = threadIdx.x;
  const int lane  = tid & 31;
  const int warp  = tid >> 5;
  const int F     = d.F;
  const int total = d.scat_tiles[d.S];
  Row* in_rows    = reinterpret_cast<Row*>(s.in);          // [2][T]
  int64_t* in_k   = reinterpret_cast<int64_t*>(s.in);      // [2][T+2]
  int64_t* in_p   = in_k + 2 * (T + 2);                    // [2][T+2]

  int prod_parent = 0;
  auto issue_tile = [&](int k) {  // thread 0 only
    const int t = blockIdx.x + k * gridDim.x;
    if (t >= total) return;
    while (d.scat_tiles[prod_parent + 1] <= t) prod_parent++;
    const int64_t beg = d.seg_begin[prod_parent] + (int64_t)(t - d.scat_tiles[prod_parent]) * T;
    int64_t end       = beg + T;
    if (end > d.seg_end[prod_parent]) end = d.seg_end[prod_parent];
    const int st = k & 1, n = (int)(end - beg);
    s.desc[st]   = TileDesc{beg, n, d.seg_parent[prod_parent]};
    if (IN_ROWS) {
      mbar_expect_tx(&s.full[st], (uint32_t)n * 16u);
      tma_load(in_rows + (size_t)st * T, d.in_rows + beg, (uint32_t)n * 16u, &s.full[st]);
    } else {
      int64_t* ks = in_k + (size_t)st * (T + 2);
      int64_t* ps = in_p + (size_t)st * (T + 2);
      const uint32_t bytes = stage_column(ks, d.in_key, beg, n, d.in_total, &s.full[st], false) +
                             stage_column(ps, d.in_pay[0], beg, n, d.in_total, &s.full[st], false);
      mbar_expect_tx(&s.full[st], bytes);
      stage_column(ks, d.in_key, beg, n, d.in_total, &s.full[st], true);
      stage_column(ps, d.in_pay[0], beg, n, d.in_total, &s.full[st], true);
    }
  };

  if (tid == kProducer) {
    mbar_init(&s.full[0], 1);
    mbar_init(&s.full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    issue_tile(0);
    issue_tile(1);
  }
  for (int i = tid; i < 2 * kMaxFanout; i += THREADS) (&s.s_cnt[0][0])[i] = 0;
  __syncthreads();

  for (int k = 0; blockIdx.x + k * (int)gridDim.x < total; k++) {
    const int st = k & 1;
    int* cnt_cur = s.s_cnt[st];
    mbar_wait(&s.full[st], (k >> 1) & 1);
    const TileDesc td = s.desc[st];
    const int tile_n  = td.n;

    // ---- rank
    int64_t key[RPT], pay[RPT];
    uint32_t brank[RPT];
    if (IN_ROWS) {
#pragma unroll
      for (int j = 0; j < RPT; j++) {
        const int r = j * THREADS + tid;
        if (r < tile_n) {
          const int4 v = *reinterpret_cast<const int4*>(in_rows + (size_t)st * T + r);
          key[j] = (int64_t)(((uint64_t)(uint32_t)v.y << 32) | (uint32_t)v.x);
          pay[j] = (int64_t)(((uint64_t)(uint32_t)v.w << 32) | (uint32_t)v.z);
        } else {
          key[j] = 0;
          pay[j] = 0;
        }
      }
    } else {
      const int64_t* ks = in_k + (size_t)st * (T + 2) + skip_of(d.in_key + td.beg);
      const int64_t* ps = in_p + (size_t)st * (T + 2) + skip_of(d.in_pay[0] + td.beg);
#pragma unroll
      for (int j = 0; j < RPT; j++) {
        const int r = j * THREADS + tid;
        key[j]      = r < tile_n ? ks[r] : 0;
        pay[j]      = r < tile_n ? ps[r] : 0;
      }
    }
#pragma unroll
    for (int j = 0; j < RPT; j++) {
      const int r = j * THREADS + tid;
      brank[j]    = 0;
      if (r < tile_n) {
        const int b = bucket_of<MODE>(key[j], d);
        brank[j]    = ((uint32_t)b << 16) | (uint32_t)atomicAdd(&cnt_cur[b], 1);
      }
    }
    __syncthreads();  // (A) tile histogram complete; the input stage has been read

    if (tid == kProducer) issue_tile(k + 2);  // refill this stage right away: the rows live in registers

    // ---- reserve + scan (thread b owns bucket b)
    const int cnt = tid < F ? cnt_cur[tid] : 0;
    unsigned long long gres = 0, gend = ~0ull;
    if (cnt) {
      gres = atomicAdd(&d.cursor[(size_t)td.parent * F + tid], (unsigned long long)cnt);
      if (d.cap_end) gend = d.cap_end[(size_t)td.parent * F + tid];
    }
    if (tid < F) s.s_cnt[st ^ 1][tid] = 0;  // the next tile's counters
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s.warp_sums[warp] = incl;
    if (LEAN && tid < F) s.s_start[tid] = incl - cnt;  // prefix inside the owning warp only
    // the previous tile's bulk copies must have read the sorted tile before it is overwritten
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    __syncthreads();  // (B)
    int excl;
    int wpre = 0;  // LEAN: lane l holds the exclusive prefix of the warp totals up to warp l
    if (LEAN) {
      const int wsum = s.warp_sums[lane];
      int winc       = wsum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
      }
      wpre = winc - wsum;
      excl = __shfl_sync(0xffffffffu, wpre, warp) + incl - cnt;
    } else {
      int wbase = lane < warp ? s.warp_sums[lane] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) wbase += __shfl_xor_sync(0xffffffffu, wbase, o);
      excl = wbase + incl - cnt;
      if (tid < F) s.s_start[tid] = excl;
      __syncthreads();  // (C)
    }

    // ---- sort: one STS.128 per row
#pragma unroll
    for (int j = 0; j < RPT; j++) {
      const int r = j * THREADS + tid;
      const int b = (int)(brank[j] >> 16);
      // bucket start = prefix of the warps before the bucket's owner + prefix inside that warp
      const int wb = LEAN ? __shfl_sync(0xffffffffu, wpre, b >> 5) : 0;  // every lane takes part
      if (r < tile_n) {
        const int pos = wb + s.s_start[b] + (int)(brank[j] & 0xffffu);
        *reinterpret_cast<int4*>(&s.srow[pos]) =
          make_int4((int)(uint32_t)(uint64_t)key[j], (int)((uint64_t)key[j] >> 32),
                    (int)(uint32_t)(uint64_t)pay[j], (int)((uint64_t)pay[j] >> 32));
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic stores -> visible to the TMA engine
    __syncthreads();  // (D) sorted tile complete

    // ---- copy-out: bucket tid's run [excl, excl+cnt) -> out_rows[gres ...); a run that would pass
    //      the bucket's capacity is dropped and its parent flagged for repair (the cursor still counts it)
    if (cnt) {
      if (gres + (unsigned long long)cnt <= gend) {
        Row* dst = (d.part_base ? d.part_base[tid >> d.part_shift] : d.out_rows) + gres;
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
                     "r"(smem_u32(&s.srow[excl])), "r"((uint32_t)cnt * 16u)
                     : "memory");
      } else {
        d.overflow[td.parent] = 1;
      }
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // writes complete before the CTA exits
}

bool use_tma_scatter()
{
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DJ_SCATTER");
    v             = (e && (e[0] == 'L' || e[0] == 'l')) ? 0 : 1;  // DJ_SCATTER=legacy disables it
  }
  return v == 1;
}

template <int MODE, bool AGG>
int launch_scatter_tma(const PassDev& dev, cudaStream_t stream)
{
  constexpr int THREADS = 1024, RPT = 4;
  const size_t smem = sizeof(ScatterTmaSmem<THREADS, RPT>);
  auto kern         = scatter_tma_kernel<MODE, AGG, THREADS, RPT>;
  DJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  {
    ProfScope prof(DJ_PROF_SCATTER, stream);
    kern<<<sm_count(), THREADS, smem, stream>>>(dev);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

bool scatter_lean()
{
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DJ_SCATTER_LEAN");
    v             = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

template <int MODE, bool IN_ROWS, bool LEAN>
int launch_scatter_rows_impl(const PassDev& dev, cudaStream_t stream, int prof_cat)
{
  constexpr int THREADS = 1024, RPT = 4;
  const size_t smem = sizeof(ScatterRowsSmem<THREADS, RPT, IN_ROWS>);
  auto kern         = scatter_rows_kernel<MODE, IN_ROWS, THREADS, RPT, LEAN>;
  DJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  {
    ProfScope prof(prof_cat, stream);
    kern<<<sm_count(), THREADS, smem, stream>>>(dev);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

template <int MODE, bool IN_ROWS>
int launch_scatter_rows(const PassDev& dev, cudaStream_t stream, int prof_cat = DJ_PROF_SCATTER)
{
  return scatter_lean() ? launch_scatter_rows_impl<MODE, IN_ROWS, true>(dev, stream, prof_cat)
                        : launch_scatter_rows_impl<MODE, IN_ROWS, false>(dev, stream, prof_cat);
}

size_t scatter_smem_bytes(int npay, int F)
{
  return (size_t)kScatterTile * 8 * (1 + npay) + (size_t)F * (8 + 4) + (size_t)kScatterTile * 2;
}

template <int MODE, int NPAY, bool AGG>
int launch_scatter(const PassDev& dev, int F, cudaStream_t stream)
{
  const size_t smem = scatter_smem_bytes(NPAY, F);
  auto kern         = scatter_kernel<MODE, NPAY, AGG>;
  DJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  DJ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kScatterThreads, smem));
  if (per_sm < 1) per_sm = 1;
  {
    ProfScope prof(DJ_PROF_SCATTER, stream);
    kern<<<sm_count() * per_sm, kScatterThreads, smem, stream>>>(dev);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

template <int MODE, int NPAY>
int launch_scatter_agg(const PassDev& dev, int F, cudaStream_t stream)
{
  return F <= 32 ? launch_scatter<MODE, NPAY, true>(dev, F, stream)
                 : launch_scatter<MODE, NPAY, false>(dev, F, stream);
}

template <int MODE>
int launch_scatter_npay(const PassDev& dev, int npay, int F, int64_t span, cudaStream_t stream)
{
  if (dev.out_rows || dev.part_base)
    return dev.in_rows ? launch_scatter_rows<MODE, true>(dev, stream) : launch_scatter_rows<MODE, false>(dev, stream);
  if (npay == 1 && span < ((int64_t)1 << 32) && use_tma_scatter())
    return F <= 32 ? launch_scatter_tma<MODE, true>(dev, stream) : launch_scatter_tma<MODE, false>(dev, stream);
  switch (npay) {
    case 1: return launch_scatter_agg<MODE, 1>(dev, F, stream);
    case 2: return launch_scatter_agg<MODE, 2>(dev, F, stream);
    case 3: return launch_scatter_agg<MODE, 3>(dev, F, stream);
  }
  set_error("partition: unsupported payload column count %d", npay);
  return DJ_ERR_ARG;
}

// ---------------------------------------------------------------- bounded passes
// Capacity of each of F child buckets of a parent holding n rows: mean + z * sigma + margin.  The
// radix bits come from local_hash (a strong mixer), so a child's size is Binomial(n, 1/F):
// sigma <= sqrt(mean).  z = 8 leaves a Gaussian tail of ~6e-16 per bucket; the constant margin
// covers the heavier tail of small means and of duplicate keys (DESIGN.md section 2).
constexpr double kCapZ       = 8.0;
constexpr int64_t kCapMargin = 32;

__host__ __device__ __forceinline__ int64_t child_capacity(int64_t n, int F)
{
  const double mean = (double)n / F;
  return (int64_t)(mean + kCapZ * sqrt(mean)) + kCapMargin;
}

// exclusive scan of one int64 per thread over a 1024-thread block
__device__ __forceinline__ int64_t block_exclusive_scan64(int64_t v, int64_t* warp_sums)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const int64_t w = warp_sums[lane];
    int64_t wi     = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    warp_sums[lane] = wi - w;
  }
  __syncthreads();
  return warp_sums[warp] + incl - v;
}

// Grid = P parents x 1024 threads.  Every CTA sums the segments' rows per parent and scans the
// parents' regions (F * capacity rows each, laid out back to back from row 0), then lays out its
// own parent: child j starts at region + j * capacity; its cursor starts there, its capacity ends
// one capacity later.  The parent's overflow flag is cleared.
__global__ void __launch_bounds__(1024)
  bucket_bases_kernel(const int64_t* seg_begin, const int64_t* seg_end, const int* seg_parent, int S, int P, int F,
                      int64_t* begin, unsigned long long* cursor, unsigned long long* cap_end, int* overflow)
{
  __shared__ unsigned long long s_rows[kMaxFanout];
  __shared__ int64_t warp_sums[32];
  __shared__ int64_t s_start, s_cap;
  const int tid = threadIdx.x, p = blockIdx.x;
  if (tid < P) s_rows[tid] = 0;
  __syncthreads();
  if (tid < S) atomicAdd(&s_rows[seg_parent[tid]], (unsigned long long)(seg_end[tid] - seg_begin[tid]));
  __syncthreads();
  const int64_t cap   = tid < P ? child_capacity((int64_t)s_rows[tid], F) : 0;
  const int64_t start = block_exclusive_scan64(cap * F, warp_sums);
  if (tid == p) {
    s_start     = start;
    s_cap       = cap;
    overflow[p] = 0;
  }
  __syncthreads();
  for (int j = tid; j < F; j += 1024) {
    const size_t b      = (size_t)p * F + j;
    const int64_t first = s_start + (int64_t)j * s_cap;
    begin[b]            = first;
    cursor[b]           = (unsigned long long)first;
    cap_end[b]          = (unsigned long long)(first + s_cap);
  }
}

__device__ unsigned long long g_radix_repairs[2];  // parents repaired per level (read_radix_repairs)

// Grid = P parents x 1024 threads (F <= 1024: one child per thread).  An overflowed parent's
// children get exact offsets inside its region: the cursors already hold exact counts (cursor -
// begin), and the region holds F * capacity >= the parent's rows.  Cursors restart at the new
// offsets, capacities end at the exact sizes.  Parents that did not overflow return at once.
__global__ void __launch_bounds__(1024) repair_bases_kernel(int F, int level, int64_t* begin, unsigned long long* cursor,
                                                            unsigned long long* cap_end, const int* overflow)
{
  __shared__ int64_t warp_sums[32];
  const int tid = threadIdx.x, p = blockIdx.x;
  if (!overflow[p]) return;
  if (tid == 0) atomicAdd(&g_radix_repairs[level], 1ull);
  const size_t b      = (size_t)p * F + tid;
  const int64_t start = begin[(size_t)p * F];
  const int64_t cnt   = tid < F ? (int64_t)cursor[b] - begin[b] : 0;
  const int64_t first = start + block_exclusive_scan64(cnt, warp_sums);  // its barriers order the reads above
  if (tid < F) {
    begin[b]   = first;
    cursor[b]  = (unsigned long long)first;
    cap_end[b] = (unsigned long long)(first + cnt);
  }
}

template <int MODE>
void launch_hist(const PassDev& dev, int grid, size_t smem, cudaStream_t stream)
{
  if (dev.in_rows)
    hist_kernel<MODE, true><<<grid, kHistThreads, smem, stream>>>(dev);
  else
    hist_kernel<MODE, false><<<grid, kHistThreads, smem, stream>>>(dev);
}

}  // namespace

// workspace: counts[P*F+1] | cursor[P*F] | seg_begin, seg_end, seg_parent[S] | hist_tiles[S+1] |
// scat_tiles[S+1] | overflow[P] | cub temp.  A bounded pass keeps its capacity ends in `counts`.
static size_t cub_scan_temp_bytes(size_t n)
{
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (unsigned long long*)nullptr,
                                (unsigned long long*)nullptr, (int)n);
  return bytes;
}

size_t pass_workspace_bytes(int P, int F, int nseg)
{
  const size_t nb = (size_t)P * F;
  const size_t S  = (size_t)(nseg > P ? nseg : P);
  size_t total    = 0;
  total += align_up((nb + 1) * 8, 256);
  total += align_up(nb * 8, 256);
  total += 2 * align_up(S * 8, 256) + align_up(S * 4, 256);
  total += 2 * align_up((S + 1) * 4, 256);
  total += align_up((size_t)P * 4, 256);
  total += align_up(cub_scan_temp_bytes(nb + 1), 256);
  return total + 1024;
}

namespace {

struct PassWs {
  unsigned long long *counts, *cursor;
  int64_t *seg_begin, *seg_end;
  int *seg_parent, *hist_tiles, *scat_tiles, *overflow;
  char* cub_temp;
  size_t cub_bytes;
};

int check_pass(const PassDesc& desc, const PassBuffers& buf, void* d_ws, size_t ws_bytes, PassWs* w, int* S_out)
{
  DJ_REQUIRE(desc.F >= 1 && desc.F <= kMaxFanout, "partition: fan-out %d out of range", desc.F);
  DJ_REQUIRE(desc.P >= 1 && desc.P <= kMaxFanout, "partition: parent count %d out of range", desc.P);
  DJ_REQUIRE(desc.mode != 1 || (desc.F & (desc.F - 1)) == 0, "radix fan-out must be a power of 2");
  DJ_REQUIRE(desc.mode != 2 || (desc.P == 1 && desc.F == desc.nparts << desc.sub_bits),
             "fused partition: F must be nparts << sub_bits");
  DJ_REQUIRE(!buf.out_rows || desc.npay == 1, "partition: row output carries exactly one payload column");
  DJ_REQUIRE(!buf.in_rows || buf.out_rows, "partition: row input needs row output");
  const bool explicit_segs = buf.d_seg_begin != nullptr;
  DJ_REQUIRE(explicit_segs || desc.P == 1 || (buf.d_parent_begin && buf.d_parent_end),
             "partition: parent ranges missing");
  const int S = explicit_segs ? buf.nseg : desc.P;
  DJ_REQUIRE(S >= 1 && S <= kMaxFanout, "partition: %d input segments (max %d)", S, kMaxFanout);
  const size_t nb = (size_t)desc.P * desc.F;
  DJ_REQUIRE(desc.align_rows == 1 || nb <= 1024, "partition: aligned buckets need P*F <= 1024");
  Arena arena(d_ws, ws_bytes);
  w->counts     = arena.take<unsigned long long>(nb + 1);
  w->cursor     = arena.take<unsigned long long>(nb);
  w->seg_begin  = arena.take<int64_t>(S);
  w->seg_end    = arena.take<int64_t>(S);
  w->seg_parent = arena.take<int>(S);
  w->hist_tiles = arena.take<int>(S + 1);
  w->scat_tiles = arena.take<int>(S + 1);
  w->overflow   = arena.take<int>(desc.P);
  w->cub_bytes  = cub_scan_temp_bytes(nb + 1);
  w->cub_temp   = arena.take<char>(w->cub_bytes);
  if (!w->counts || !w->cursor || !w->seg_begin || !w->seg_end || !w->seg_parent || !w->hist_tiles ||
      !w->scat_tiles || !w->overflow || !w->cub_temp) {
    set_error("partition pass: workspace too small (%zu bytes given)", ws_bytes);
    return DJ_ERR_WORKSPACE;
  }
  *S_out = S;
  return DJ_OK;
}

int launch_plan(const PassBuffers& buf, int S, const PassWs& w, cudaStream_t stream)
{
  plan_kernel<<<1, 1024, 0, stream>>>(buf.d_parent_begin, buf.d_parent_end, buf.d_seg_begin, buf.d_seg_end,
                                      buf.d_seg_parent, buf.nrows, S, kScatterTile, w.seg_begin, w.seg_end,
                                      w.seg_parent, w.hist_tiles, w.scat_tiles, nullptr);
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

PassDev make_dev(const PassDesc& desc, const PassBuffers& buf, int S, const PassWs& w)
{
  PassDev dev{};
  dev.in_key  = buf.in_key;
  dev.out_key = buf.out_key;
  for (int c = 0; c < desc.npay; c++) {
    dev.in_pay[c]  = buf.in_pay[c];
    dev.out_pay[c] = buf.out_pay[c];
  }
  dev.in_rows    = buf.in_rows;
  dev.out_rows   = buf.out_rows;
  dev.part_base  = nullptr;
  dev.part_shift = 0;
  dev.in_total   = buf.nrows;
  dev.seg_begin  = w.seg_begin;
  dev.seg_end    = w.seg_end;
  dev.seg_parent = w.seg_parent;
  dev.counts     = w.counts;
  dev.cursor     = w.cursor;
  dev.hist_tiles = w.hist_tiles;
  dev.scat_tiles = w.scat_tiles;
  dev.S          = S;
  dev.P          = desc.P;
  dev.F          = desc.F;
  dev.seed       = desc.seed;
  dev.hash_id    = desc.hash_id;
  dev.shift      = desc.shift;
  dev.pow2       = desc.mode == 2 ? (desc.nparts & (desc.nparts - 1)) == 0 : (desc.F & (desc.F - 1)) == 0;
  dev.nparts     = desc.nparts;
  dev.sub_bits   = desc.sub_bits;
  return dev;
}

}  // namespace

int pass_histogram(const PassDesc& desc, const PassBuffers& buf, void* d_ws, size_t ws_bytes,
                   cudaStream_t stream, PassState* state)
{
  PassWs w;
  int S  = 0;
  int rc = check_pass(desc, buf, d_ws, ws_bytes, &w, &S);
  if (rc) return rc;
  const size_t nb = (size_t)desc.P * desc.F;
  DJ_CUDA_TRY(cudaMemsetAsync(w.counts, 0, (nb + 1) * 8, stream));
  if ((rc = launch_plan(buf, S, w, stream))) return rc;
  const PassDev dev = make_dev(desc, buf, S, w);

  const int hist_grid = sm_count() * 4;
  const size_t hsmem  = (size_t)desc.F * sizeof(int);
  {
    ProfScope prof(DJ_PROF_HIST, stream);
    if (desc.mode == 0)
      launch_hist<0>(dev, hist_grid, hsmem, stream);
    else if (desc.mode == 1)
      launch_hist<1>(dev, hist_grid, hsmem, stream);
    else
      launch_hist<2>(dev, hist_grid, hsmem, stream);
  }
  DJ_LAUNCH_CHECK();

  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    if (desc.align_rows > 1) {
      aligned_offsets_kernel<<<1, 1024, 0, stream>>>(w.counts, (int)nb, desc.mode == 2 ? 1 << desc.sub_bits : 1,
                                                     desc.align_rows, buf.d_child_off, buf.d_child_cnt);
      count_launch(1);
    } else {
      DJ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(w.cub_temp, w.cub_bytes, w.counts,
                                                (unsigned long long*)buf.d_child_off, (int)(nb + 1),
                                                stream));
      count_launch(2);
    }
    DJ_CUDA_TRY(cudaMemcpyAsync(w.cursor, buf.d_child_off, nb * 8, cudaMemcpyDeviceToDevice, stream));
  }
  state->dev  = dev;
  state->mode = desc.mode;
  state->npay = desc.npay;
  // 32-bit destination offsets in the SoA TMA kernel: input rows + worst-case padding must fit
  state->span = buf.nrows + (int64_t)nb * desc.align_rows;
  return DJ_OK;
}

int pass_scatter(const PassState& st, cudaStream_t stream)
{
  if (st.mode == 0) return launch_scatter_npay<0>(st.dev, st.npay, st.dev.F, st.span, stream);
  if (st.mode == 1) return launch_scatter_npay<1>(st.dev, st.npay, st.dev.F, st.span, stream);
  return launch_scatter_npay<2>(st.dev, st.npay, st.dev.F, st.span, stream);
}

int run_partition_pass(const PassDesc& desc, const PassBuffers& buf, void* d_ws, size_t ws_bytes,
                       cudaStream_t stream)
{
  PassState st;
  int rc = pass_histogram(desc, buf, d_ws, ws_bytes, stream, &st);
  if (rc) return rc;
  return pass_scatter(st, stream);
}

// Sum over parents of F * child_capacity(n_p, F) <= sum of (n_p + z * sqrt(F * n_p) + F * (margin + 1))
// (the +1 absorbs rounding), and sum of sqrt(n_p) <= sqrt(P * nrows) by concavity.
int64_t bounded_pass_rows(int64_t nrows, int P, int F)
{
  const double nb = (double)P * F;
  return nrows + (int64_t)std::ceil(kCapZ * std::sqrt(nb * (double)nrows)) + (int64_t)nb * (kCapMargin + 1);
}

int run_bounded_pass(const PassDesc& desc, const PassBuffers& buf, int level, void* d_ws, size_t ws_bytes,
                     cudaStream_t stream)
{
  DJ_REQUIRE(desc.mode == 1 && buf.out_rows && buf.d_child_off && buf.d_child_end && level >= 0 && level < 2,
             "partition: bounded passes are row-output radix passes");
  PassWs w;
  int S  = 0;
  int rc = check_pass(desc, buf, d_ws, ws_bytes, &w, &S);
  if (rc) return rc;
  if ((rc = launch_plan(buf, S, w, stream))) return rc;
  auto* cursor  = reinterpret_cast<unsigned long long*>(buf.d_child_end);
  auto* cap_end = w.counts;
  {
    ProfScope prof(DJ_PROF_HIST, stream);
    bucket_bases_kernel<<<desc.P, 1024, 0, stream>>>(w.seg_begin, w.seg_end, w.seg_parent, S, desc.P, desc.F,
                                                     buf.d_child_off, cursor, cap_end, w.overflow);
  }
  DJ_LAUNCH_CHECK();
  PassDev dev  = make_dev(desc, buf, S, w);
  dev.cursor   = cursor;
  dev.cap_end  = cap_end;
  dev.overflow = w.overflow;
  rc = buf.in_rows ? launch_scatter_rows<1, true>(dev, stream) : launch_scatter_rows<1, false>(dev, stream);
  if (rc) return rc;

  // repair, always enqueued: exact offsets for overflowed parents, their segments re-planned in
  // place (every other segment emptied), and the scatter again over those segments only
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    repair_bases_kernel<<<desc.P, 1024, 0, stream>>>(desc.F, level, buf.d_child_off, cursor, cap_end, w.overflow);
    count_launch(1);
    plan_kernel<<<1, 1024, 0, stream>>>(nullptr, nullptr, w.seg_begin, w.seg_end, w.seg_parent, buf.nrows, S,
                                        kScatterTile, w.seg_begin, w.seg_end, w.seg_parent, w.hist_tiles,
                                        w.scat_tiles, w.overflow);
  }
  DJ_LAUNCH_CHECK();
  return buf.in_rows ? launch_scatter_rows<1, true>(dev, stream, DJ_PROF_OTHER)
                     : launch_scatter_rows<1, false>(dev, stream, DJ_PROF_OTHER);
}

int read_radix_repairs(int64_t out[2])
{
  unsigned long long v[2] = {0, 0};
  DJ_CUDA_TRY(cudaDeviceSynchronize());
  DJ_CUDA_TRY(cudaMemcpyFromSymbol(v, g_radix_repairs, sizeof(v)));
  const unsigned long long zero[2] = {0, 0};
  DJ_CUDA_TRY(cudaMemcpyToSymbol(g_radix_repairs, zero, sizeof(zero)));
  out[0] = (int64_t)v[0];
  out[1] = (int64_t)v[1];
  return DJ_OK;
}

const void* partition_module_kernel() { return (const void*)plan_kernel; }

}  // namespace dj
