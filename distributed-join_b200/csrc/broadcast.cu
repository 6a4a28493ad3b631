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
// Build: init, insert (claim + count, each row remembers its slot and rank in its key's run), CUB
// exclusive scan of the counts, place.  Semi and anti joins need the key set only and stop after insert.
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

// KIND 0: inner join, DJ_JOIN_LEFT_SEMI, DJ_JOIN_LEFT_ANTI, DJ_JOIN_LEFT_OUTER.
// Per tile: every thread probes its rows and counts its output rows; rows of long runs go to a list.
// One block scan places the short rows, warp 0 scans the list, and ONE atomicAdd reserves the tile's
// output.  Short rows are staged in shared memory in output order and leave as coalesced column runs;
// each long run is written by one warp, 32 consecutive rows per store.
// (At least 4 CTAs per SM: without that bound ptxas holds the semi / anti kernels to 40 registers and
// spills.)
template <int KIND>
__global__ void __launch_bounds__(kProbeThreads, 4) bcast_probe_kernel(ProbeDev d)
{
  constexpr bool kPairs = KIND == 0 || KIND == DJ_JOIN_LEFT_OUTER;  // emits right payloads
  constexpr bool kOuter = KIND == DJ_JOIN_LEFT_OUTER;
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

size_t broadcast_table_bytes(int64_t nright)
{
  Arena a(reinterpret_cast<void*>(4096), ~(size_t)0 >> 1);  // sizes only: any non-null aligned base
  take_table(a, nright);
  return a.used;
}

int broadcast_hash_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* rk,
                        const int64_t* rp, int64_t nr, int64_t* const out[4], uint8_t* out_sides,
                        int64_t out_capacity, int64_t* d_out_count, Arena& arena, cudaStream_t stream)
{
  DJ_REQUIRE(nr <= DJ_BROADCAST_TABLE_MAX_ROWS, "broadcast join: %lld right rows exceed the hash table's %d",
             (long long)nr, (int)DJ_BROADCAST_TABLE_MAX_ROWS);
  const Table t = take_table(arena, nr);
  if (!t.ok) {
    set_error("broadcast join: workspace too small for the hash table");
    return DJ_ERR_WORKSPACE;
  }
  const bool pairs = kind == 0 || kind == DJ_JOIN_LEFT_OUTER;
  const int build_grid = (int)std::min<int64_t>(std::max<int64_t>((nr + kBuildThreads - 1) / kBuildThreads, 1),
                                                (int64_t)sm_count() * 8);
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    bcast_init_kernel<<<std::min<int>((t.nslots + kBuildThreads) / kBuildThreads, sm_count() * 8), kBuildThreads, 0,
                        stream>>>(t.keys, t.cnt, t.nslots);
  }
  DJ_LAUNCH_CHECK();
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
  if (nl == 0) return DJ_OK;
  ProbeDev d{};
  d.lk = lk; d.lp = lp; d.nl = nl;
  d.keys = t.keys; d.cnt = t.cnt; d.start = t.start; d.run_pay = t.run_pay;
  d.mask = t.nslots - 1;
  for (int c = 0; c < 4; c++) d.out[c] = out[c];
  d.sides        = out_sides;
  d.out_capacity = out_capacity;
  d.out_count    = (unsigned long long*)d_out_count;
  switch (kind) {
    case 0: return launch_probe<0>(d, stream);
    case DJ_JOIN_LEFT_SEMI: return launch_probe<DJ_JOIN_LEFT_SEMI>(d, stream);
    case DJ_JOIN_LEFT_ANTI: return launch_probe<DJ_JOIN_LEFT_ANTI>(d, stream);
    case DJ_JOIN_LEFT_OUTER: return launch_probe<DJ_JOIN_LEFT_OUTER>(d, stream);
  }
  set_error("broadcast join: unknown join kind %d", kind);
  return DJ_ERR_ARG;
}

const void* broadcast_module_kernel() { return (const void*)bcast_probe_kernel<0>; }

}  // namespace dj
