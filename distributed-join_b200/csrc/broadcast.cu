// broadcast.cu -- the broadcast join's local join: a left table probed where it lies, against a hash
// table of the gathered right table (include/dj_b200.h, dj_broadcast_join_i64).
//
// The repartitioned joins radix-partition both sides so that every bucket's build side fits in shared
// memory.  When the whole right table is small, its hash table fits in L2 instead, and the left table
// needs no partitioning at all: it is read once, coalesced, and every row looks its key up in the table.
//
// Table: open addressing with linear probing over 2^k >= 2 * nright slots (at most half filled), ONE
// slot per DISTINCT key.  With one slot per row, a key repeated 100k times would be a 100k-slot
// cluster that every probe landing near it walks.  Arrays (each separate, so that a probe reads only
// the 8-byte keys until it hits):
//   keys[nslots]       the slot's key, kEmptyKey while free (claimed with a 64-bit CAS)
//   cnt[nslots + 1]    right rows with that key; cnt[nslots] is the side slot of the rows whose key IS
//                      kEmptyKey, which can occupy no regular slot because every int64 is a valid key
//   start[nslots + 1]  (inner / left outer) exclusive scan of cnt: the key's run in run_pay
//   run_pay[nright]    (inner / left outer) the right payloads, grouped into one contiguous run per key
//   mark[nslots + 1]   (full outer) set once a left row of this rank has hit the slot
// Build: init, insert (claim + count, each row remembers its slot and rank in its key's run), CUB
// exclusive scan of the counts, place.  Semi and anti joins need the key set only and stop after insert.
//
// The broadcast full outer join (dj_broadcast_full_outer_join_i64) needs one more thing from the local
// join: which gathered right rows this rank's left rows matched, as one bit per gathered row in gathered
// order (`matched`), because that is the only form in which the ranks' verdicts can be ORed: slot order
// depends on CAS timing and the radix path's bucket order on atomics.  The hash path marks slots in the
// probe and maps the marks to rows through row_slot; the radix path joins (gathered key, gathered row
// index) with the kJoinFullOuterMark kernel, maps its build-row bits to rows through that index, and
// puts the real right payloads into its pairs afterwards.  The exchange of the bits and the emit of the
// rows no rank matched follow in comm.cu (broadcast_join) and broadcast_emit_unmatched_right below.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "dj_device.cuh"
#include "dj_internal.h"

namespace dj {
namespace {

constexpr int64_t kEmptyKey = INT64_MIN;  // a free slot's key; rows with this key live in the side slot
constexpr int kBuildThreads = 256;
// probe: a CTA takes tiles of kTile left rows, kRowsPerThread per thread at a stride of kProbeThreads
// (every load instruction of a warp covers 32 consecutive rows)
constexpr int kProbeThreads = 256, kRowsPerThread = 4, kTile = kProbeThreads * kRowsPerThread;
// a left row matching more right rows than this is a "long run": it is not staged, a whole warp
// writes it straight out (a hot right key must not serialise one lane)
constexpr int kLongRun = 32;
// output rows staged per round; short rows of a tile beyond it take further rounds
constexpr int kStage = 1024;
constexpr uint32_t kMiss = 0xFFFFFFFFu;  // run start of a left row without a match (no run starts there)
static_assert((int64_t)DJ_BROADCAST_TABLE_MAX_ROWS * kTile < ((int64_t)1 << 31),
              "a tile's long-run rows are counted in 32 bits");

__device__ __forceinline__ uint32_t table_hash(int64_t key) { return local_hash_i64(key); }

__global__ void __launch_bounds__(kBuildThreads) bcast_init_kernel(int64_t* keys, uint32_t* cnt, uint32_t nslots)
{
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= nslots; i += gridDim.x * blockDim.x) {
    if (i < nslots) keys[i] = kEmptyKey;
    cnt[i] = 0;
  }
}

// Claims (or finds) every right row's slot and counts the row into it.  row_slot / row_pos (nullptr for
// semi / anti) receive the slot and the row's rank inside its key's run.
__global__ void __launch_bounds__(kBuildThreads) bcast_insert_kernel(const int64_t* __restrict__ rk, int64_t nr,
                                                                     int64_t* keys, uint32_t* cnt, uint32_t mask,
                                                                     uint32_t* row_slot, uint32_t* row_pos)
{
  const uint32_t nslots = mask + 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nr; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = rk[i];
    uint32_t s      = nslots;
    if (k != kEmptyKey) {
      s = table_hash(k) & mask;
      while (true) {
        // keys only ever go from kEmptyKey to their final value, so a stale read can only be a
        // kEmptyKey, and the CAS then returns the truth
        const int64_t cur = keys[s];
        if (cur == k) break;
        if (cur == kEmptyKey) {
          const int64_t prev = (int64_t)atomicCAS(reinterpret_cast<unsigned long long*>(keys + s),
                                                  (unsigned long long)kEmptyKey, (unsigned long long)k);
          if (prev == kEmptyKey || prev == k) break;
        }
        s = (s + 1) & mask;
      }
    }
    const uint32_t pos = atomicAdd(cnt + s, 1u);
    if (row_slot) {
      row_slot[i] = s;
      row_pos[i]  = pos;
    }
  }
}

__global__ void __launch_bounds__(kBuildThreads) bcast_place_kernel(const int64_t* __restrict__ rp, int64_t nr,
                                                                    const uint32_t* __restrict__ row_slot,
                                                                    const uint32_t* __restrict__ row_pos,
                                                                    const uint32_t* __restrict__ start,
                                                                    int64_t* run_pay)
{
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nr; i += (int64_t)gridDim.x * blockDim.x)
    run_pay[start[row_slot[i]] + row_pos[i]] = rp[i];
}

struct ProbeDev {
  const int64_t* lk;
  const int64_t* lp;
  int64_t nl;
  const int64_t* keys;
  const uint32_t* cnt;
  const uint32_t* start;
  const int64_t* run_pay;
  uint32_t mask;
  int64_t* out[4];
  uint8_t* sides;
  int64_t out_capacity;
  unsigned long long* out_count;
  uint8_t* mark;  // full outer: [nslots + 1] bytes, set for every slot a left row hits
};

// slot of `k`, or -1 when the table does not hold it
__device__ __forceinline__ int64_t find_slot(const ProbeDev& d, int64_t k)
{
  if (k == kEmptyKey) return __ldg(d.cnt + d.mask + 1) ? (int64_t)d.mask + 1 : -1;
  uint32_t s = table_hash(k) & d.mask;
  while (true) {
    const int64_t cur = __ldg(d.keys + s);
    if (cur == k) return s;
    if (cur == kEmptyKey) return -1;
    s = (s + 1) & d.mask;
  }
}

// KIND 0: inner join, DJ_JOIN_LEFT_SEMI, DJ_JOIN_LEFT_ANTI, DJ_JOIN_LEFT_OUTER.  DJ_JOIN_FULL_OUTER
// writes what the left outer join writes and also marks every slot it hits (d.mark): a plain store, and
// only where a plain load still sees the mark clear, so that the rows of a hot key do not all store.
// Per tile: every thread probes its rows and counts its output rows; rows of long runs go to a list.
// One block scan places the short rows, warp 0 scans the list, and ONE atomicAdd reserves the tile's
// output.  Short rows are staged in shared memory in output order and leave as coalesced column runs;
// each long run is written by one warp, 32 consecutive rows per store.
// (At least 4 CTAs per SM: without that bound ptxas holds the semi / anti kernels to 40 registers and
// spills.)
template <int KIND>
__global__ void __launch_bounds__(kProbeThreads, 4) bcast_probe_kernel(ProbeDev d)
{
  constexpr bool kPairs = KIND == 0 || KIND == DJ_JOIN_LEFT_OUTER || KIND == DJ_JOIN_FULL_OUTER;  // right payloads
  constexpr bool kOuter = KIND == DJ_JOIN_LEFT_OUTER || KIND == DJ_JOIN_FULL_OUTER;
  constexpr bool kMarks = KIND == DJ_JOIN_FULL_OUTER;
  __shared__ int64_t s_lk[kStage], s_lp[kStage], s_rp[kPairs ? kStage : 1];
  __shared__ uint8_t s_side[kOuter ? kStage : 1];
  constexpr int kLongMax = kPairs ? kTile : 1;  // every row of a tile may be a long run
  __shared__ int s_long_row[kLongMax], s_long_off[kLongMax];
  __shared__ uint32_t s_long_cnt[kLongMax], s_long_start[kLongMax];
  __shared__ int s_warp[33];
  __shared__ int s_nlong;
  __shared__ unsigned long long s_base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  for (int64_t t0 = (int64_t)blockIdx.x * kTile; t0 < d.nl; t0 += (int64_t)gridDim.x * kTile) {
    if (tid == 0) s_nlong = 0;
    __syncthreads();  // also: the previous tile is done with every shared array
    int64_t key[kRowsPerThread], pay[kRowsPerThread];
    uint32_t n[kRowsPerThread], rs[kRowsPerThread];  // short output rows of the row, its run start
    int nshort = 0;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; j++) {
      const int64_t r = t0 + j * kProbeThreads + tid;
      n[j]            = 0;
      rs[j]           = kMiss;
      key[j] = pay[j] = 0;
      if (r < d.nl) {
        key[j]             = __ldcs(d.lk + r);  // streamed once: keep it out of the table's way in L2
        pay[j]             = __ldcs(d.lp + r);
        const int64_t slot = find_slot(d, key[j]);
        if (kMarks && slot >= 0 && !d.mark[slot]) d.mark[slot] = 1;
        if (KIND == DJ_JOIN_LEFT_SEMI) n[j] = slot >= 0;
        if (KIND == DJ_JOIN_LEFT_ANTI) n[j] = slot < 0;
        if (kPairs) {
          const uint32_t c = slot >= 0 ? __ldg(d.cnt + slot) : 0;
          n[j]             = kOuter && c == 0 ? 1 : c;
          if (c) rs[j] = __ldg(d.start + slot);  // a miss keeps kMiss
          if (c > (uint32_t)kLongRun) {
            const int e     = atomicAdd(&s_nlong, 1);
            s_long_row[e]   = j * kProbeThreads + tid;
            s_long_cnt[e]   = c;
            s_long_start[e] = rs[j];
            n[j]            = 0;
          }
        }
      }
      nshort += (int)n[j];
    }
    const int off        = block_exclusive_scan<kProbeThreads>(nshort, s_warp);  // two barriers: s_nlong is final
    const int short_rows = s_warp[32];
    // read before the reservation barrier below: thread 0 resets s_nlong for the next tile only after
    // passing that barrier, i.e. after every thread has read it
    const int nlong = kPairs ? s_nlong : 0;
    if (warp == 0) {
      // the long runs' output offsets (in list order), then the tile's one reservation
      const int per   = (nlong + 31) / 32;
      int sum         = 0;
      for (int e = lane * per; e < min(nlong, (lane + 1) * per); e++) sum += (int)s_long_cnt[e];
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      int at = incl - sum;
      for (int e = lane * per; e < min(nlong, (lane + 1) * per); e++) {
        s_long_off[e] = at;
        at += (int)s_long_cnt[e];
      }
      const int long_rows = __shfl_sync(0xffffffffu, incl, 31);
      if (lane == 0) {
        const unsigned long long total = (unsigned long long)short_rows + (unsigned long long)long_rows;
        s_base = total ? atomicAdd(d.out_count, total) : 0;
      }
    }
    __syncthreads();
    const int64_t base = (int64_t)s_base;
    // short rows, kStage output rows per round
    for (int c0 = 0; c0 < short_rows && base + c0 < d.out_capacity; c0 += kStage) {
      int o = off - c0;  // this thread's next row, relative to the round
#pragma unroll
      for (int j = 0; j < kRowsPerThread; j++) {
        for (uint32_t k = 0; k < n[j]; k++, o++) {
          if (o < 0 || o >= kStage) continue;
          s_lk[o] = key[j];
          s_lp[o] = pay[j];
          if (kPairs) {
            const bool hit = rs[j] != kMiss;
            s_rp[o]        = hit ? __ldg(d.run_pay + rs[j] + k) : 0;
            if (kOuter) s_side[o] = hit ? (DJ_SIDE_LEFT | DJ_SIDE_RIGHT) : DJ_SIDE_LEFT;
          }
        }
      }
      __syncthreads();
      const int m = min(kStage, short_rows - c0);
      for (int i = tid; i < m; i += kProbeThreads) {
        const int64_t g = base + c0 + i;
        if (g >= d.out_capacity) break;
        d.out[0][g] = s_lk[i];
        d.out[1][g] = s_lp[i];
        if (kPairs) {
          const bool hit = !kOuter || s_side[i] != DJ_SIDE_LEFT;
          d.out[2][g]    = hit ? s_lk[i] : 0;
          d.out[3][g]    = s_rp[i];
          if (kOuter) d.sides[g] = s_side[i];
        }
      }
      __syncthreads();  // the stage is rewritten by the next round
    }
    if (kPairs) {
      // long runs: one warp per run, 32 consecutive output rows per store
      for (int e = warp; e < nlong; e += kProbeThreads / 32) {
        const int64_t r  = t0 + s_long_row[e];
        const int64_t k  = __ldg(d.lk + r), p = __ldg(d.lp + r);
        const int64_t g0 = base + short_rows + s_long_off[e];
        const uint32_t c = s_long_cnt[e], st = s_long_start[e];
        for (uint32_t i = lane; i < c; i += 32) {
          const int64_t g = g0 + i;
          if (g >= d.out_capacity) break;
          d.out[0][g] = k;
          d.out[1][g] = p;
          d.out[2][g] = k;
          d.out[3][g] = __ldg(d.run_pay + st + i);
          if (kOuter) d.sides[g] = DJ_SIDE_LEFT | DJ_SIDE_RIGHT;
        }
      }
    }
  }
}

template <int KIND>
int launch_probe(const ProbeDev& d, cudaStream_t stream)
{
  // resident CTAs per SM (fixed block size and shared memory), found once; rank threads of a local group
  // may get here at the same time, and a function-local static is initialised exactly once
  static const int per_sm = [] {
    int n = 0;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, bcast_probe_kernel<KIND>, kProbeThreads, 0) ==
               cudaSuccess
             ? std::max(n, 1)
             : 0;
  }();
  if (!per_sm) {
    set_error("broadcast join: cannot query the probe kernel's occupancy");
    return DJ_ERR_CUDA;
  }
  const int64_t tiles = (d.nl + kTile - 1) / kTile;
  const int grid      = (int)std::min<int64_t>(tiles, (int64_t)sm_count() * per_sm);
  {
    ProfScope prof(DJ_PROF_JOIN, stream);
    bcast_probe_kernel<KIND><<<grid, kProbeThreads, 0, stream>>>(d);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

// Full outer, hash path: matched[g >> 5] bit g & 31 = the mark of gathered row g's slot.  One warp covers
// 32 consecutive rows and writes their word.
__global__ void __launch_bounds__(kBuildThreads) bcast_matched_bits_kernel(const uint32_t* __restrict__ row_slot,
                                                                           const uint8_t* __restrict__ mark,
                                                                           int64_t nr, uint32_t* matched)
{
  const int lane = threadIdx.x & 31;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i - lane < nr;
       i += (int64_t)gridDim.x * blockDim.x) {
    const bool hit   = i < nr && mark[row_slot[i]];
    const uint32_t w = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) matched[i >> 5] = w;
  }
}

__global__ void __launch_bounds__(kBuildThreads) bcast_iota_kernel(int64_t* out, int64_t n)
{
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = i;
}

// Full outer, radix path: the build side's payloads are gathered row indices, so every prepared build
// row whose bit the kJoinFullOuterMark join set names its gathered row.  Buckets are walked as
// emit_unmatched_build_kernel walks them (the gaps between buckets hold stale rows).
__global__ void __launch_bounds__(kBuildThreads) bcast_translate_marks_kernel(const Row* __restrict__ rows,
                                                                              const int64_t* __restrict__ bbeg,
                                                                              const int64_t* __restrict__ bend,
                                                                              int nbuckets,
                                                                              const uint32_t* __restrict__ bits,
                                                                              uint32_t* matched)
{
  for (int b = blockIdx.x; b < nbuckets; b += gridDim.x) {
    const int64_t b1 = bend[b];
    for (int64_t r = bbeg[b] + threadIdx.x; r < b1; r += blockDim.x) {
      if (!((bits[r >> 5] >> (r & 31)) & 1u)) continue;
      const int64_t g = rows[r].pay;
      atomicOr(matched + (g >> 5), 1u << (g & 31));
    }
  }
}

// Full outer, radix path: the pairs carry the gathered row index as their right payload; the output
// rows below min(count, capacity) with both sides get the real payload grp[g].
__global__ void __launch_bounds__(kBuildThreads) bcast_fix_pair_payloads_kernel(const uint8_t* __restrict__ sides,
                                                                                int64_t* rp_out,
                                                                                const int64_t* __restrict__ grp,
                                                                                const unsigned long long* count,
                                                                                int64_t out_capacity)
{
  const int64_t n = min((int64_t)*count, out_capacity);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (sides[i] == (DJ_SIDE_LEFT | DJ_SIDE_RIGHT)) rp_out[i] = __ldg(grp + rp_out[i]);
}

// Full outer: appends every row i of this rank's right slice (rk, rp)[n] whose bit is clear in every
// inbox row as (0, 0, key, payload) with sides DJ_SIDE_RIGHT, at the running count.  Row i's bit is bit
// (bit0 + i) & 31 of word (bit0 + i) >> 5 of each of the `rows` inbox rows (row_words words apart): the
// slice starts at gathered row `before`, and the words every rank sent start at word before >> 5, so
// bit0 = before & 31.  A tile of kTile rows reserves its output with ONE atomicAdd, as
// emit_unmatched_build_kernel does; every row is counted, none is written at or past the capacity.
__global__ void __launch_bounds__(kProbeThreads) bcast_emit_unmatched_right_kernel(
  const int64_t* __restrict__ rk, const int64_t* __restrict__ rp, int64_t n, const uint32_t* __restrict__ inbox,
  int rows, int64_t row_words, int bit0, int64_t* null_key, int64_t* null_pay, int64_t* out_key, int64_t* out_pay,
  uint8_t* out_sides, int64_t out_capacity, unsigned long long* out_count)
{
  constexpr int kRuns = kTile / 32;  // (warp, step) runs of 32 rows in a tile
  __shared__ unsigned long long run_base[kRuns];
  __shared__ int run_cnt[kRuns];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t t0 = (int64_t)blockIdx.x * kTile; t0 < n; t0 += (int64_t)gridDim.x * kTile) {
    unsigned lone[kRowsPerThread];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; j++) {
      const int64_t i = t0 + j * kProbeThreads + threadIdx.x;
      bool mine       = false;
      if (i < n) {
        const int64_t b = bit0 + i;
        uint32_t w      = 0;
        for (int r = 0; r < rows; r++) w |= __ldg(inbox + r * row_words + (b >> 5));
        mine = !((w >> (b & 31)) & 1u);
      }
      lone[j] = __ballot_sync(0xffffffffu, mine);
      if (lane == 0) run_cnt[j * (kProbeThreads / 32) + warp] = __popc(lone[j]);
    }
    __syncthreads();
    if (warp == 0) {
      // exclusive scan of the kRuns counts (kRuns / 32 per lane), one reservation for the tile
      int c[kRuns / 32], sum = 0;
#pragma unroll
      for (int i = 0; i < kRuns / 32; i++) {
        c[i] = run_cnt[lane * (kRuns / 32) + i];
        sum += c[i];
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int total      = __shfl_sync(0xffffffffu, incl, 31);
      unsigned long long g = 0;
      if (lane == 0 && total) g = atomicAdd(out_count, (unsigned long long)total);
      g = __shfl_sync(0xffffffffu, g, 0) + (unsigned long long)(incl - sum);
#pragma unroll
      for (int i = 0; i < kRuns / 32; i++) {
        run_base[lane * (kRuns / 32) + i] = g;
        g += c[i];
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kRowsPerThread; j++) {
      if (!((lone[j] >> lane) & 1u)) continue;
      const int64_t g = (int64_t)run_base[j * (kProbeThreads / 32) + warp] + __popc(lone[j] & lanemask_lt());
      if (g < out_capacity) {
        const int64_t i = t0 + j * kProbeThreads + threadIdx.x;
        null_key[g]     = 0;
        null_pay[g]     = 0;
        out_key[g]      = __ldg(rk + i);
        out_pay[g]      = __ldg(rp + i);
        out_sides[g]    = DJ_SIDE_RIGHT;
      }
    }
    // the next tile writes run_base only past its first barrier, i.e. after every thread's reads above
  }
}

// blocks of kBuildThreads for a grid-stride loop over `threads` threads
int grid_for(int64_t threads)
{
  return (int)std::min<int64_t>(std::max<int64_t>((threads + kBuildThreads - 1) / kBuildThreads, 1),
                                (int64_t)sm_count() * 8);
}

uint32_t table_slots(int64_t nright)
{
  uint32_t s = 64;
  while ((int64_t)s < 2 * nright) s <<= 1;
  return s;
}

size_t scan_temp_bytes(uint32_t n)
{
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
  return bytes;
}

// The table's arrays, taken from `a` in one fixed order (broadcast_table_bytes replays it).
struct Table {
  uint32_t nslots;
  int64_t* keys;
  uint32_t *cnt, *start, *row_slot, *row_pos;
  int64_t* run_pay;
  char* scan_temp;
  size_t scan_bytes;
  bool ok;
};
Table take_table(Arena& a, int64_t nr)
{
  Table t{};
  t.nslots     = table_slots(nr);
  t.keys       = a.take<int64_t>(t.nslots);
  t.cnt        = a.take<uint32_t>((size_t)t.nslots + 1);
  t.start      = a.take<uint32_t>((size_t)t.nslots + 1);
  t.row_slot   = a.take<uint32_t>((size_t)nr);
  t.row_pos    = a.take<uint32_t>((size_t)nr);
  t.run_pay    = a.take<int64_t>((size_t)nr);
  t.scan_bytes = scan_temp_bytes(t.nslots + 1);
  t.scan_temp  = a.take<char>(t.scan_bytes);
  t.ok         = t.keys && t.cnt && t.start && t.row_slot && t.row_pos && t.run_pay && t.scan_temp;
  return t;
}

}  // namespace

size_t broadcast_table_bytes(int64_t nright, int kind)
{
  Arena a(reinterpret_cast<void*>(4096), ~(size_t)0 >> 1);  // sizes only: any non-null aligned base
  const Table t = take_table(a, nright);
  if (kind == DJ_JOIN_FULL_OUTER) a.take<uint8_t>((size_t)t.nslots + 1);  // the slot marks
  return a.used;
}

int broadcast_hash_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* rk,
                        const int64_t* rp, int64_t nr, int64_t* const out[4], uint8_t* out_sides,
                        int64_t out_capacity, int64_t* d_out_count, Arena& arena, cudaStream_t stream,
                        uint32_t* d_matched)
{
  DJ_REQUIRE(nr <= DJ_BROADCAST_TABLE_MAX_ROWS, "broadcast join: %lld right rows exceed the hash table's %d",
             (long long)nr, (int)DJ_BROADCAST_TABLE_MAX_ROWS);
  const bool full = kind == DJ_JOIN_FULL_OUTER;
  const Table t   = take_table(arena, nr);
  uint8_t* mark   = full ? arena.take<uint8_t>((size_t)t.nslots + 1) : nullptr;
  if (!t.ok || (full && !mark)) {
    set_error("broadcast join: workspace too small for the hash table");
    return DJ_ERR_WORKSPACE;
  }
  const bool pairs = kind == 0 || kind == DJ_JOIN_LEFT_OUTER || full;
  const int build_grid = (int)std::min<int64_t>(std::max<int64_t>((nr + kBuildThreads - 1) / kBuildThreads, 1),
                                                (int64_t)sm_count() * 8);
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    bcast_init_kernel<<<std::min<int>((t.nslots + kBuildThreads) / kBuildThreads, sm_count() * 8), kBuildThreads, 0,
                        stream>>>(t.keys, t.cnt, t.nslots);
  }
  DJ_LAUNCH_CHECK();
  if (full) DJ_CUDA_TRY(cudaMemsetAsync(mark, 0, (size_t)t.nslots + 1, stream));
  if (nr > 0) {
    {
      ProfScope prof(DJ_PROF_OTHER, stream);
      bcast_insert_kernel<<<build_grid, kBuildThreads, 0, stream>>>(rk, nr, t.keys, t.cnt, t.nslots - 1,
                                                                    pairs ? t.row_slot : nullptr, t.row_pos);
    }
    DJ_LAUNCH_CHECK();
    if (pairs) {
      size_t bytes = t.scan_bytes;
      {
        ProfScope prof(DJ_PROF_OTHER, stream);
        DJ_CUDA_TRY(cub::DeviceScan::ExclusiveSum(t.scan_temp, bytes, t.cnt, t.start, (int)t.nslots + 1, stream));
      }
      count_launch();
      {
        ProfScope prof(DJ_PROF_OTHER, stream);
        bcast_place_kernel<<<build_grid, kBuildThreads, 0, stream>>>(rp, nr, t.row_slot, t.row_pos, t.start,
                                                                     t.run_pay);
      }
      DJ_LAUNCH_CHECK();
    }
  }
  if (nl > 0) {
    ProbeDev d{};
    d.lk = lk; d.lp = lp; d.nl = nl;
    d.keys = t.keys; d.cnt = t.cnt; d.start = t.start; d.run_pay = t.run_pay;
    d.mask = t.nslots - 1;
    for (int c = 0; c < 4; c++) d.out[c] = out[c];
    d.sides        = out_sides;
    d.out_capacity = out_capacity;
    d.out_count    = (unsigned long long*)d_out_count;
    d.mark         = mark;
    int rc         = DJ_ERR_ARG;
    switch (kind) {
      case 0: rc = launch_probe<0>(d, stream); break;
      case DJ_JOIN_LEFT_SEMI: rc = launch_probe<DJ_JOIN_LEFT_SEMI>(d, stream); break;
      case DJ_JOIN_LEFT_ANTI: rc = launch_probe<DJ_JOIN_LEFT_ANTI>(d, stream); break;
      case DJ_JOIN_LEFT_OUTER: rc = launch_probe<DJ_JOIN_LEFT_OUTER>(d, stream); break;
      case DJ_JOIN_FULL_OUTER: rc = launch_probe<DJ_JOIN_FULL_OUTER>(d, stream); break;
      default: set_error("broadcast join: unknown join kind %d", kind);
    }
    if (rc) return rc;
  }
  if (full && nr > 0) {
    // every gathered row's mark, read through its slot (the marks are zero without left rows)
    {
      ProfScope prof(DJ_PROF_OTHER, stream);
      bcast_matched_bits_kernel<<<grid_for((nr + 31) / 32 * 32), kBuildThreads, 0, stream>>>(t.row_slot, mark, nr,
                                                                                             d_matched);
    }
    DJ_LAUNCH_CHECK();
  }
  return DJ_OK;
}

size_t broadcast_radix_mark_bytes(int64_t nl, int64_t nr)
{
  return local_join_workspace(DJ_JOIN_FULL_OUTER, nr, nl) + filter_bits_bytes(nr, join_plan(DJ_JOIN_FULL_OUTER, nr)) +
         align_up((size_t)nr * 8, 256) + 256;
}

int broadcast_radix_mark_join(const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* grk,
                              const int64_t* grp, int64_t nr, int64_t* const out[4], uint8_t* out_sides,
                              int64_t out_capacity, int64_t* d_out_count, uint32_t* d_matched, Arena& arena,
                              cudaStream_t stream)
{
  DJ_CUDA_TRY(cudaMemsetAsync(d_matched, 0, (size_t)(nr + 31) / 32 * 4, stream));
  if (nl == 0 || nr == 0) return DJ_OK;
  auto ws_too_small = [] {
    set_error("broadcast join: workspace too small for the radix-partitioned join");
    return DJ_ERR_WORKSPACE;
  };
  // the build side is (gathered key, gathered row index): every prepared build row knows its row
  int64_t* iota = arena.take<int64_t>((size_t)nr);
  if (!iota) return ws_too_small();
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    bcast_iota_kernel<<<grid_for(nr), kBuildThreads, 0, stream>>>(iota, nr);
  }
  DJ_LAUNCH_CHECK();
  const RadixPlan plan = join_plan(DJ_JOIN_FULL_OUTER, nr);
  const TableInput tb{grk, iota, nullptr, nr, nullptr, nullptr, 0}, tp{lk, lp, nullptr, nl, nullptr, nullptr, 0};
  PreparedSide sb{}, sp{};
  int rc = prepare_side(tb, plan, &sb, arena, stream);
  if (rc) return rc;
  rc = prepare_side(tp, plan, &sp, arena, stream);
  if (rc) return rc;
  const size_t words = (size_t)(sb.cap_rows + 31) / 32;
  uint32_t* bits     = arena.take<uint32_t>(words);
  if (!bits) return ws_too_small();
  DJ_CUDA_TRY(cudaMemsetAsync(bits, 0, words * 4, stream));
  rc = join_prepared(kJoinFullOuterMark, sb, sp, plan, out, out_sides, out_capacity, d_out_count, true, arena, stream,
                     bits);
  if (rc) return rc;
  // the marks are set whether or not a pair fitted the output, so `matched` is exact past the capacity
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    bcast_translate_marks_kernel<<<std::min(plan.nbuckets, sm_count() * 8), kBuildThreads, 0, stream>>>(
      sb.rows, sb.d_begin, sb.d_end, plan.nbuckets, bits, d_matched);
  }
  DJ_LAUNCH_CHECK();
  if (out_capacity > 0) {
    {
      ProfScope prof(DJ_PROF_OTHER, stream);
      bcast_fix_pair_payloads_kernel<<<sm_count() * 4, kBuildThreads, 0, stream>>>(
        out_sides, out[3], grp, (const unsigned long long*)d_out_count, out_capacity);
    }
    DJ_LAUNCH_CHECK();
  }
  return DJ_OK;
}

int broadcast_emit_unmatched_right(const int64_t* rk, const int64_t* rp, int64_t n, const uint32_t* inbox, int rows,
                                   int64_t row_words, int bit0, int64_t* const out[4], uint8_t* out_sides,
                                   int64_t out_capacity, int64_t* d_out_count, cudaStream_t stream)
{
  if (n == 0) return DJ_OK;
  const int grid = (int)std::min<int64_t>((n + kTile - 1) / kTile, (int64_t)sm_count() * 8);
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    bcast_emit_unmatched_right_kernel<<<grid, kProbeThreads, 0, stream>>>(
      rk, rp, n, inbox, rows, row_words, bit0, out[0], out[1], out[2], out[3], out_sides, out_capacity,
      (unsigned long long*)d_out_count);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

const void* broadcast_module_kernel() { return (const void*)bcast_probe_kernel<0>; }

}  // namespace dj
