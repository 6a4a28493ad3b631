// join.cu -- shared-memory open-addressing hash build + probe for sm_90a (H100).
//
// Replaces cudf::inner_join as called by local_join_helper (src/distributed_join.cpp:71-83).
// Both tables arrive radix-partitioned (partition.cu, mode 1) into buckets whose build side
// fits one CTA's shared-memory table.  One persistent CTA per SM (31 consumer warps + 1
// producer warp) walks a contiguous range of buckets:
//
//   producer warp   one elected lane streams every bucket's rows HBM -> shared memory with TMA
//                   bulk copies (cp.async.bulk + mbarrier complete_tx): one build-chunk stage
//                   and a ring of probe-chunk stages, refilled as soon as consumers release them,
//                   so global-memory latency never sits on the consumers' critical path;
//   consumer warps  1. insert the staged build rows (16-byte (key, payload) rows, one TMA copy per
//                      chunk) into a linear-probing table of 32-bit (fingerprint, row) slots claimed
//                      with atomicCAS -- the staged rows are the row store, no key value is reserved
//                      as "empty"; two tables ping-pong so the next one is cleared off the critical
//                      path,
//                   2. probe one staged row per lane; matches are compacted with __ballot_sync /
//                      popc into a shared-memory output tile,
//                   3. flush full output tiles with ONE global atomicAdd per tile and coalesced
//                      stores; the atomic's round trip is hidden behind the next round of probing
//                      (three tiles rotate), and batch results land in one output so no
//                      cudf::concatenate is needed afterwards.
// Multimap semantics: probing continues past a hit until an empty slot.  Build buckets larger
// than one chunk (skew / duplicates) are processed chunk by chunk, re-streaming the probe side.
//
// Left semi / left anti joins (KIND = DJ_JOIN_LEFT_SEMI / DJ_JOIN_LEFT_ANTI) run the same kernel
// with the right table as the build side and the left table as the probe side.  A probe stops at
// its first key match and emits the probe row itself, (key, payload), at most once: semi on a
// match, anti when the cluster ends without one.  When a bucket's build side spans several build
// jobs, a row's verdict is kept across the jobs in one bit per prepared probe row (d.probe_bits,
// zeroed before the launch): semi emits a row when its atomicOr finds the bit clear, anti sets
// bits in every job but the last and emits, in the last, the rows with neither a bit nor a match.
// The jobs of a bucket run in order in one CTA, and the consumer barrier between two jobs orders
// the bit updates.  An anti join also runs one (empty) build job for a bucket whose build side is
// empty, so that its probe rows are all emitted.
//
// Left / full outer joins (KIND = DJ_JOIN_LEFT_OUTER / DJ_JOIN_FULL_OUTER) also build on the right
// table.  The probe loop is the inner join's multimap loop; each lane also remembers whether its row
// matched in this job, and the anti join's bit rule decides, in a bucket's last job, which probe rows
// matched nothing: those are emitted once with an absent build side.  A full outer join keeps one bit
// per staged build row in shared memory (set on every match); every probe row of the bucket streams
// past every build job, so at the end of a job the build rows with a clear bit are exactly the right
// rows without a match, and they are emitted with an absent probe side.  Output tiles of these kinds
// carry a sides byte next to the four columns (bit 0: probe / left row present, bit 1: build / right
// row present); absent columns are written as 0.
//
// A full outer join whose left table arrives in several launches (the streamed host entry joins it
// chunk by chunk) cannot use that per-job verdict: a right row is unmatched only if no chunk matched
// it.  KIND = kJoinFullOuterMark is a left outer join that keeps the same shared-memory bits and, at
// the end of a job, ORs them into one global bit per row position of the build side (d.build_bits,
// zeroed once per call).  After the last chunk emit_unmatched_build_kernel appends the build rows
// whose bit is still clear.
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "dj_device.cuh"
#include "dj_internal.h"

namespace dj {

namespace {

// Compile-time shape of one CTA.  Two shapes are built: A = one 1024-thread CTA per SM for
// ~1.5K-row buckets, B = two 512-thread CTAs per SM for ~0.75K-row buckets.
template <int THREADS, int SLOTS, int BUILD_CHUNK, int TARGET_ROWS, int PROBE_STAGES, int OUT_ROWS>
struct JoinCfg {
  static constexpr int kThreads     = THREADS;
  static constexpr int kConsumers   = THREADS - 32;
  static constexpr int kConsWarps   = kConsumers / 32;
  static constexpr int kSlots       = SLOTS;        // 32-bit slots per table (power of 2)
  static constexpr int kBuildChunk  = BUILD_CHUNK;  // max build rows per table (<= 2048)
  static constexpr int kTargetRows  = TARGET_ROWS;  // planned average build rows per bucket
  static constexpr int kProbeChunk  = kConsumers;   // one probe row per consumer thread and round
  static constexpr int kProbeStages = PROBE_STAGES;
  static constexpr int kOutRows     = OUT_ROWS;     // rows per output tile
};
using CfgA = JoinCfg<1024, 8192, 1792, 1536, 2, 576>;
using CfgB = JoinCfg<512, 4096, 1024, 768, 2, 256>;

constexpr int kOutTiles    = 3;    // filling / atomicAdd in flight / draining
constexpr int kDescBuckets = 128;  // bucket descriptors cached per refill

struct JoinDev {
  const Row* build;
  const int64_t *bbeg, *bend;  // bucket b = rows [bbeg[b], bend[b]) of build
  const Row* probe;
  const int64_t *pbeg, *pend;
  int nbuckets;
  int64_t* out[4];
  int64_t out_capacity;
  unsigned long long* out_count;
  uint32_t* probe_bits;  // semi / anti / outer: one bit per row of `probe` (multi-job buckets only)
  uint8_t* out_sides;    // outer joins: DJ_SIDE_* bits of every output row
  uint32_t* build_bits;  // kMark: one bit per row position of `build`, set for matched rows
};

constexpr int kInner = 0, kSemi = DJ_JOIN_LEFT_SEMI, kAnti = DJ_JOIN_LEFT_ANTI;
constexpr int kLeftOuter = DJ_JOIN_LEFT_OUTER, kFullOuter = DJ_JOIN_FULL_OUTER, kMark = kJoinFullOuterMark;
// sides byte of an outer join's output row, in the kernel's (build, probe) terms: the probe side is
// the left table, the build side the right one
constexpr uint8_t kSideProbe = DJ_SIDE_LEFT, kSideBuild = DJ_SIDE_RIGHT;

__host__ __device__ constexpr bool is_outer(int kind)
{
  return kind == kLeftOuter || kind == kFullOuter || kind == kMark;
}
// kinds that keep a "matched" bit per staged build row
__host__ __device__ constexpr bool marks_build(int kind) { return kind == kFullOuter || kind == kMark; }

template <class C>
struct __align__(128) JoinSmem {
  uint32_t slots[2][C::kSlots];
  Row brow[2][C::kBuildChunk];
  Row prow[C::kProbeStages][C::kProbeChunk];
  int64_t sout[kOutTiles][4][C::kOutRows];
  int64_t dbb[kDescBuckets], dbe[kDescBuckets];  // cached bucket ranges, build side
  int64_t dpb[kDescBuckets], dpe[kDescBuckets];  // probe side
  unsigned long long full_build[2], empty_build[2];
  unsigned long long full_probe[C::kProbeStages], empty_probe[C::kProbeStages];
  unsigned long long sbase[kOutTiles];
  int scnt[kOutTiles];
};

// Outer joins: the output tiles' sides bytes, and (full outer, mark) one "matched" bit per staged
// build row of each of the two tables.
template <class C>
struct __align__(128) OuterJoinSmem : JoinSmem<C> {
  uint8_t ssides[kOutTiles][C::kOutRows];
  uint32_t bmatch[2][C::kBuildChunk / 32];
};

template <class C, int KIND>
using JoinSmemOf = std::conditional_t<is_outer(KIND), OuterJoinSmem<C>, JoinSmem<C>>;

template <int N>
__device__ __forceinline__ void consumer_sync()
{
  asm volatile("bar.sync 1, %0;" ::"n"(N) : "memory");
}

// Build jobs of the cached descriptor block: (bucket, build chunk) pairs whose bucket is
// non-empty on both sides (anti, left outer: on the probe side; full outer: on either side).
// Every thread walks them identically.
template <int KIND, class S>
__device__ __forceinline__ int next_valid_bucket(const S& s, int lb, int nd)
{
  if constexpr (KIND == kAnti || KIND == kLeftOuter || KIND == kMark) {
    while (lb < nd && s.dpe[lb] == s.dpb[lb]) lb++;
  } else if constexpr (KIND == kFullOuter) {
    while (lb < nd && s.dbe[lb] == s.dbb[lb] && s.dpe[lb] == s.dpb[lb]) lb++;
  } else {
    while (lb < nd && (s.dbe[lb] == s.dbb[lb] || s.dpe[lb] == s.dpb[lb])) lb++;
  }
  return lb;
}

// Slot word: bit 31 = occupied, bits 30..11 = 20-bit key fingerprint, bits 10..0 = build row.
__device__ __forceinline__ uint32_t slot_tag(uint32_t h) { return 0x100000u | (h >> 12); }

// Outer joins: every lane with `emit` set appends the row (bk, bp, pk, pv, sides) to output tile
// `cur`; once the tile is full, the warp reserves its own run of the output and stores the rest
// directly.  Called by all 32 lanes of a warp.
template <class C>
__device__ __forceinline__ void emit_outer_row(OuterJoinSmem<C>& s, const JoinDev& d, int cur, int lane, bool emit,
                                               int64_t bk, int64_t bp, int64_t pk, int64_t pv, uint8_t sides)
{
  const unsigned m = __ballot_sync(0xffffffffu, emit);
  if (m == 0) return;
  const int leader = __ffs(m) - 1;
  int obase        = 0;
  if (lane == leader) {
    obase = atomicAdd(&s.scnt[cur], __popc(m));
    if (obase >= C::kOutRows) atomicSub(&s.scnt[cur], __popc(m));  // a full tile stays full (see inner)
  }
  obase            = __shfl_sync(0xffffffffu, obase, leader);
  const int pos    = obase + __popc(m & lanemask_lt());
  const bool spill = emit && pos >= C::kOutRows;
  if (emit && !spill) {
    s.sout[cur][0][pos] = bk;
    s.sout[cur][1][pos] = bp;
    s.sout[cur][2][pos] = pk;
    s.sout[cur][3][pos] = pv;
    s.ssides[cur][pos]  = sides;
  }
  const unsigned ms = __ballot_sync(0xffffffffu, spill);
  if (ms) {
    const int sl         = __ffs(ms) - 1;
    unsigned long long g = 0;
    if (lane == sl) g = atomicAdd(d.out_count, (unsigned long long)__popc(ms));
    g = __shfl_sync(0xffffffffu, g, sl);
    if (spill) {
      const int64_t gi = (int64_t)g + __popc(ms & lanemask_lt());
      if (gi < d.out_capacity) {
        d.out[0][gi]     = bk;
        d.out[1][gi]     = bp;
        d.out[2][gi]     = pk;
        d.out[3][gi]     = pv;
        d.out_sides[gi]  = sides;
      }
    }
  }
}

template <class C, int KIND>
__global__ void __launch_bounds__(C::kThreads, 1) bucket_join_kernel(JoinDev d)
{
  using Smem = JoinSmemOf<C, KIND>;
  constexpr int kConsumers = C::kConsumers;
  constexpr bool kOuter    = is_outer(KIND);
  // a bucket with probe rows but no build rows still runs one (empty) build job
  constexpr bool kEmptyJob = KIND == kAnti || kOuter;
  constexpr int kCols      = (KIND == kSemi || KIND == kAnti) ? 2 : 4;  // output columns
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& s        = *reinterpret_cast<Smem*>(smem_raw);
  const int tid  = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const bool is_producer = warp == C::kConsWarps;

  if (tid == 0) {
    for (int i = 0; i < 2; i++) {
      mbar_init(&s.full_build[i], 1);
      mbar_init(&s.empty_build[i], C::kConsWarps);
    }
    for (int i = 0; i < C::kProbeStages; i++) {
      mbar_init(&s.full_probe[i], 1);
      mbar_init(&s.empty_probe[i], C::kConsWarps);
    }
    for (int i = 0; i < kOutTiles; i++) s.scnt[i] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < 2 * C::kSlots; i += C::kThreads) (&s.slots[0][0])[i] = 0;
  if constexpr (marks_build(KIND))
    for (int i = tid; i < 2 * (C::kBuildChunk / 32); i += C::kThreads) (&s.bmatch[0][0])[i] = 0;
  __syncthreads();

  // contiguous bucket range of this CTA
  const int lo = (int)((int64_t)d.nbuckets * blockIdx.x / gridDim.x);
  const int hi = (int)((int64_t)d.nbuckets * (blockIdx.x + 1) / gridDim.x);

  uint32_t q = 0;  // probe-job ordinal (stage = q % kProbeStages)
  uint32_t u = 0;  // build-job ordinal (stage = table = u & 1)
  // Output tiles rotate filling -> pending (its atomicAdd is in flight during the next build
  // job) -> draining (copied out while a third tile already fills) -> free.
  int cur = 0, pend_tile = 0, pend_n = 0;
  unsigned long long pend_base_reg = 0;  // thread 0 only

  for (int base = lo; base < hi; base += kDescBuckets) {
    const int nd = min(kDescBuckets, hi - base);
    __syncthreads();  // everyone is done with the previous descriptors
    for (int i = tid; i < nd; i += C::kThreads) {
      s.dbb[i] = d.bbeg[base + i];
      s.dbe[i] = d.bend[base + i];
      s.dpb[i] = d.pbeg[base + i];
      s.dpe[i] = d.pend[base + i];
    }
    __syncthreads();

    if (is_producer) {
      // ------------------------------------------------------------ producer (one lane)
      if (lane == 0) {
        for (int lb = next_valid_bucket<KIND>(s, 0, nd); lb < nd; lb = next_valid_bucket<KIND>(s, lb + 1, nd)) {
          const int64_t b0 = s.dbb[lb], b1 = s.dbe[lb], p0 = s.dpb[lb], p1 = s.dpe[lb];
          for (int64_t c0 = b0; c0 < b1 || (kEmptyJob && c0 == b0); c0 += C::kBuildChunk) {
            {
              const int bs = u & 1;
              const int n  = (int)min((int64_t)C::kBuildChunk, b1 - c0);  // 0 for an empty build job
              mbar_wait(&s.empty_build[bs], ((u >> 1) & 1) ^ 1);
              mbar_expect_tx(&s.full_build[bs], (uint32_t)n * 16u);
              if (!kEmptyJob || n > 0) tma_load(s.brow[bs], d.build + c0, (uint32_t)n * 16u, &s.full_build[bs]);
              u++;
            }
            for (int64_t r0 = p0; r0 < p1; r0 += C::kProbeChunk) {
              const int st = q % C::kProbeStages;
              const int n  = (int)min((int64_t)C::kProbeChunk, p1 - r0);
              mbar_wait(&s.empty_probe[st], ((q / C::kProbeStages) & 1) ^ 1);
              mbar_expect_tx(&s.full_probe[st], (uint32_t)n * 16u);
              tma_load(s.prow[st], d.probe + r0, (uint32_t)n * 16u, &s.full_probe[st]);
              q++;
            }
          }
        }
      }
      __syncwarp();  // reconverge before the CTA-wide barrier at the top of the loop
    } else {
      // ------------------------------------------------------------ consumers
      for (int lb = next_valid_bucket<KIND>(s, 0, nd); lb < nd; lb = next_valid_bucket<KIND>(s, lb + 1, nd)) {
        const int64_t b0 = s.dbb[lb], b1 = s.dbe[lb], p0 = s.dpb[lb], p1 = s.dpe[lb];
        // semi / anti / outer: does this bucket's build side span several jobs, and is this its last job
        const bool multi = KIND != kInner && b1 - b0 > C::kBuildChunk;
        for (int64_t c0 = b0; c0 < b1 || (kEmptyJob && c0 == b0); c0 += C::kBuildChunk) {
          const bool last = c0 + C::kBuildChunk >= b1;
          // ---- build: fingerprint + row index into a 32-bit slot claimed with atomicCAS; the
          //      staged rows themselves are the row store (no copy)
          const int bs = u & 1;
          const int nb = (int)min((int64_t)C::kBuildChunk, b1 - c0);
          uint32_t* slots     = s.slots[bs];
          const Row* brow     = s.brow[bs];
          mbar_wait(&s.full_build[bs], (u >> 1) & 1);
          for (int r = tid; r < nb; r += kConsumers) {
            const uint32_t h = slot_hash_i64(brow[r].key);
            const uint32_t e = (slot_tag(h) << 11) | (uint32_t)r;
            uint32_t slot    = h & (C::kSlots - 1);
            while (atomicCAS(&slots[slot], 0u, e) != 0u) slot = (slot + 1) & (C::kSlots - 1);
          }
          // the other table was last probed two build jobs ago: clear it for the next job
          {
            uint4* other = reinterpret_cast<uint4*>(s.slots[bs ^ 1]);
            for (int i = tid; i < C::kSlots / 4; i += kConsumers) other[i] = make_uint4(0, 0, 0, 0);
            if constexpr (KIND == kFullOuter)
              for (int i = tid; i < C::kBuildChunk / 32; i += kConsumers) s.bmatch[bs ^ 1][i] = 0;
          }
          consumer_sync<kConsumers>();  // table complete

          // ---- probe: every warp streams its 32 rows of each staged chunk at its own pace
          for (int64_t r0 = p0; r0 < p1; r0 += C::kProbeChunk) {
            const int st = q % C::kProbeStages;
            const int np = (int)min((int64_t)C::kProbeChunk, p1 - r0);
            mbar_wait(&s.full_probe[st], (q / C::kProbeStages) & 1);
            bool alive = tid < np;
            int64_t k = 0, v = 0;
            if (alive) {
              const int4 pr = *reinterpret_cast<const int4*>(&s.prow[st][tid]);
              k = (int64_t)(((uint64_t)(uint32_t)pr.y << 32) | (uint32_t)pr.x);
              v = (int64_t)(((uint64_t)(uint32_t)pr.w << 32) | (uint32_t)pr.z);
            }
            // Release the stage only once every lane's row has LANDED in registers: neither __syncwarp
            // nor the arrive waits for an outstanding shared-memory load, and the producer's next TMA
            // copy into this stage (async proxy) is not ordered after it, so it could overwrite a row
            // a lane had not read yet (that lane then probed a row of the chunk two ahead twice).  The
            // reduction consumes the loaded registers, and the arrive depends on its (always nonzero)
            // result.
            const unsigned landed =
              __reduce_and_sync(0xffffffffu, (uint32_t)((uint64_t)k ^ ((uint64_t)k >> 32) ^ (uint64_t)v ^
                                                        ((uint64_t)v >> 32)) | 1u);
            if (lane == 0 && landed) mbar_arrive(&s.empty_probe[st]);
            q++;

            const uint32_t h    = slot_hash_i64(k);
            const uint32_t want = slot_tag(h);
            uint32_t slot       = h & (C::kSlots - 1);
            if constexpr (kOuter) {
              // outer: the inner join's multimap walk, remembering whether this row matched at all
              const bool valid = alive;
              bool matched     = false;
              while (true) {
                bool found = false;
                int idx    = 0;
                if (alive) {
                  while (true) {
                    const uint32_t e = slots[slot];
                    if (e == 0u) {
                      alive = false;
                      break;
                    }
                    if ((e >> 11) == want) {
                      idx = (int)(e & 0x7ffu);
                      if (brow[idx].key == k) {
                        found = true;
                        break;
                      }
                    }
                    slot = (slot + 1) & (C::kSlots - 1);
                  }
                }
                if (!__any_sync(0xffffffffu, found)) break;
                int64_t bpay = 0;
                if (found) {
                  matched = true;
                  bpay    = brow[idx].pay;
                  if constexpr (marks_build(KIND)) {
                    uint32_t* w      = &s.bmatch[bs][idx >> 5];
                    const uint32_t b = 1u << (idx & 31);
                    if (!(*w & b)) atomicOr(w, b);
                  }
                }
                emit_outer_row<C>(s, d, cur, lane, found, k, bpay, k, v, kSideBuild | kSideProbe);
                if (found) slot = (slot + 1) & (C::kSlots - 1);  // multimap: scan past the hit
              }
              // the anti join's rule: a row is unmatched when no job of its bucket matched it
              const int64_t prow_at = r0 + tid;
              uint32_t* word        = d.probe_bits + (prow_at >> 5);
              const uint32_t bit    = 1u << (prow_at & 31);
              if (multi && matched && !last) atomicOr(word, bit);
              const bool lone = valid && !matched && last && (!multi || !(__ldcg(word) & bit));
              emit_outer_row<C>(s, d, cur, lane, lone, 0, 0, k, v, kSideProbe);
              continue;
            }
            if constexpr (KIND == kSemi || KIND == kAnti) {
              // semi / anti: walk to the first key match or to the end of the cluster
              bool found = false;
              if (alive) {
                while (true) {
                  const uint32_t e = slots[slot];
                  if (e == 0u) break;
                  if ((e >> 11) == want && brow[e & 0x7ffu].key == k) {
                    found = true;
                    break;
                  }
                  slot = (slot + 1) & (C::kSlots - 1);
                }
              }
              const int64_t prow_at = r0 + tid;  // position of this row in the prepared probe side
              uint32_t* word        = d.probe_bits + (prow_at >> 5);
              const uint32_t bit    = 1u << (prow_at & 31);
              bool emit;
              if constexpr (KIND == kSemi) {
                emit = found && (!multi || !(atomicOr(word, bit) & bit));
              } else {
                if (multi && found && !last) atomicOr(word, bit);
                // L2 read: the bits were set by atomics, and L1 may hold the word from an earlier bucket
                emit = alive && !found && last && (!multi || !(__ldcg(word) & bit));
              }
              const unsigned m = __ballot_sync(0xffffffffu, emit);
              if (m) {
                const int leader = __ffs(m) - 1;
                int obase        = 0;
                if (lane == leader) {
                  obase = atomicAdd(&s.scnt[cur], __popc(m));
                  if (obase >= C::kOutRows) atomicSub(&s.scnt[cur], __popc(m));
                }
                obase            = __shfl_sync(0xffffffffu, obase, leader);
                const int pos    = obase + __popc(m & lanemask_lt());
                const bool spill = emit && pos >= C::kOutRows;
                if (emit && !spill) {
                  s.sout[cur][0][pos] = k;
                  s.sout[cur][1][pos] = v;
                }
                const unsigned ms = __ballot_sync(0xffffffffu, spill);
                if (ms) {
                  const int sl = __ffs(ms) - 1;
                  unsigned long long g = 0;
                  if (lane == sl) g = atomicAdd(d.out_count, (unsigned long long)__popc(ms));
                  g = __shfl_sync(0xffffffffu, g, sl);
                  if (spill) {
                    const int64_t gi = (int64_t)g + __popc(ms & lanemask_lt());
                    if (gi < d.out_capacity) {
                      d.out[0][gi] = k;
                      d.out[1][gi] = v;
                    }
                  }
                }
              }
              continue;
            }
            while (true) {
              bool found = false;
              int idx    = 0;
              if (alive) {
                // walk to the next fingerprint+key match or to the end of the cluster
                while (true) {
                  const uint32_t e = slots[slot];
                  if (e == 0u) {
                    alive = false;
                    break;
                  }
                  if ((e >> 11) == want) {
                    idx = (int)(e & 0x7ffu);
                    if (brow[idx].key == k) {
                      found = true;
                      break;
                    }
                  }
                  slot = (slot + 1) & (C::kSlots - 1);
                }
              }
              const unsigned m = __ballot_sync(0xffffffffu, found);
              if (m == 0) break;
              const int leader = __ffs(m) - 1;
              int obase        = 0;
              if (lane == leader) {
                obase = atomicAdd(&s.scnt[cur], __popc(m));
                // a full tile stays "full": spilled matches are counted by the global counter below, so
                // pull the tile counter back and keep it from ever wrapping (hot keys: > 2^31 matches)
                if (obase >= C::kOutRows) atomicSub(&s.scnt[cur], __popc(m));
              }
              obase         = __shfl_sync(0xffffffffu, obase, leader);
              const int pos = obase + __popc(m & lanemask_lt());
              const bool spill = found && pos >= C::kOutRows;
              if (found && !spill) {
                s.sout[cur][0][pos] = k;
                s.sout[cur][1][pos] = brow[idx].pay;
                s.sout[cur][2][pos] = k;
                s.sout[cur][3][pos] = v;
              }
              // tile full (high selectivity / duplicates): the warp reserves its own run of
              // the output with one atomicAdd and stores it directly
              const unsigned ms = __ballot_sync(0xffffffffu, spill);
              if (ms) {
                const int sl = __ffs(ms) - 1;
                unsigned long long g = 0;
                if (lane == sl) g = atomicAdd(d.out_count, (unsigned long long)__popc(ms));
                g = __shfl_sync(0xffffffffu, g, sl);
                if (spill) {
                  const int64_t gi = (int64_t)g + __popc(ms & lanemask_lt());
                  if (gi < d.out_capacity) {
                    d.out[0][gi] = k;
                    d.out[1][gi] = brow[idx].pay;
                    d.out[2][gi] = k;
                    d.out[3][gi] = v;
                  }
                }
              }
              if (found) slot = (slot + 1) & (C::kSlots - 1);  // multimap: scan past the hit
            }
          }

          // ---- end of build job: table and row store are released, output tiles rotate
          if (tid == 0 && pend_n) s.sbase[pend_tile] = pend_base_reg;
          consumer_sync<kConsumers>();
          if constexpr (KIND == kFullOuter) {
            // every probe row of the bucket has passed this job: its build rows with a clear bit match
            // no left row.  They are read from the row store and appended to tile `cur`, so the store
            // is released and the tile handed over only after a second barrier.
            for (int r0 = tid - lane; r0 < nb; r0 += kConsumers) {
              const int r     = r0 + lane;
              const bool lone = r < nb && !((s.bmatch[bs][r >> 5] >> (r & 31)) & 1u);
              int64_t bk = 0, bp = 0;
              if (lone) {
                bk = brow[r].key;
                bp = brow[r].pay;
              }
              emit_outer_row<C>(s, d, cur, lane, lone, bk, bp, 0, 0, kSideBuild);
            }
            consumer_sync<kConsumers>();
          }
          if constexpr (KIND == kMark) {
            // This job's matched bits move to the global array at the job's row position c0.  Thread i
            // owns word i of bmatch[bs] from this barrier on: the job's atomicOrs all precede the
            // barrier above, nothing sets a bit of bmatch[bs] again before the probe phase of job
            // u + 2, and every thread reaches that phase only through job u + 1's two barriers, which
            // this thread passes after the flush.  So a plain read and a plain store of 0 are
            // ordered, no second barrier is needed, and the build phase does not clear bmatch for
            // this kind.  Buckets start at any row, so a word straddles two global words, which
            // neighbouring jobs (of this or another CTA) may share: atomicOr.
            if (tid < C::kBuildChunk / 32) {
              const uint32_t w = s.bmatch[bs][tid];
              if (w) {
                s.bmatch[bs][tid] = 0;
                const int64_t at  = c0 + 32 * tid;
                uint32_t* g       = d.build_bits + (at >> 5);
                const int sh      = (int)(at & 31);
                atomicOr(g, w << sh);
                if (sh && (w >> (32 - sh))) atomicOr(g + 1, w >> (32 - sh));
              }
            }
          }
          if (lane == 0) mbar_arrive(&s.empty_build[bs]);
          if (pend_n) {
            // copy out the tile whose atomicAdd was issued one build job ago (latency hidden);
            // it stays untouched until the job after next, when every thread is past here
            const int64_t gb = (int64_t)s.sbase[pend_tile];
#pragma unroll
            for (int c = 0; c < kCols; c++)
              for (int i = tid; i < pend_n; i += kConsumers)
                if (gb + i < d.out_capacity) d.out[c][gb + i] = s.sout[pend_tile][c][i];
            if constexpr (kOuter)
              for (int i = tid; i < pend_n; i += kConsumers)
                if (gb + i < d.out_capacity) d.out_sides[gb + i] = s.ssides[pend_tile][i];
            if (tid == 0) s.scnt[pend_tile] = 0;
            pend_n = 0;
          }
          int n_out = s.scnt[cur];
          if (n_out > 0) {
            if (n_out > C::kOutRows) n_out = C::kOutRows;
            if (tid == 0) pend_base_reg = atomicAdd(d.out_count, (unsigned long long)n_out);
            pend_n    = n_out;
            pend_tile = cur;
            cur       = cur + 1 == kOutTiles ? 0 : cur + 1;
          }
          u++;
        }
      }
    }
  }

  // ---- drain the pending tile (the current one is empty: every job hands its tile over)
  if (!is_producer) {
    if (tid == 0 && pend_n) s.sbase[pend_tile] = pend_base_reg;
    consumer_sync<kConsumers>();
    if (pend_n) {
      const int64_t gb = (int64_t)s.sbase[pend_tile];
#pragma unroll
      for (int c = 0; c < kCols; c++)
        for (int i = tid; i < pend_n; i += kConsumers)
          if (gb + i < d.out_capacity) d.out[c][gb + i] = s.sout[pend_tile][c][i];
      if constexpr (kOuter)
        for (int i = tid; i < pend_n; i += kConsumers)
          if (gb + i < d.out_capacity) d.out_sides[gb + i] = s.ssides[pend_tile][i];
    }
  }
}

int join_shape()
{
  static int shape = -1;
  if (shape < 0) {
    const char* e = getenv("DJ_JOIN_SHAPE");
    shape         = (e && (e[0] == 'B' || e[0] == 'b')) ? 1 : 0;
  }
  return shape;
}

template <class C, int KIND>
int launch_join(const JoinDev& d, int ctas_per_sm, cudaStream_t stream)
{
  const size_t smem = sizeof(JoinSmemOf<C, KIND>);
  auto kern         = bucket_join_kernel<C, KIND>;
  DJ_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = sm_count() * ctas_per_sm;
  if (grid > d.nbuckets) grid = d.nbuckets;
  {
    ProfScope prof(DJ_PROF_JOIN, stream);
    kern<<<grid, C::kThreads, smem, stream>>>(d);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

template <class C>
int launch_join_kind(const JoinDev& d, int kind, int ctas_per_sm, cudaStream_t stream)
{
  return kind == kSemi        ? launch_join<C, kSemi>(d, ctas_per_sm, stream)
         : kind == kAnti      ? launch_join<C, kAnti>(d, ctas_per_sm, stream)
         : kind == kLeftOuter ? launch_join<C, kLeftOuter>(d, ctas_per_sm, stream)
         : kind == kFullOuter ? launch_join<C, kFullOuter>(d, ctas_per_sm, stream)
         : kind == kMark      ? launch_join<C, kMark>(d, ctas_per_sm, stream)
                              : launch_join<C, kInner>(d, ctas_per_sm, stream);
}

// Appends the rows of segments [sb[i], se[i]) of `rows` (blockIdx.y = segment) to (out_key, out_pay)
// at the running count: an anti or outer join's rows whose other side is empty in this batch.  Outer
// joins also zero the absent side's columns (null_key, null_pay) and set the rows' sides byte.
constexpr int kAppendChunk = 4096;  // rows per output reservation

__global__ void __launch_bounds__(256) append_rows_kernel(const Row* rows, const int64_t* sb, const int64_t* se,
                                                          int64_t* out_key, int64_t* out_pay, int64_t* null_key,
                                                          int64_t* null_pay, uint8_t* out_sides, uint8_t sides,
                                                          int64_t out_capacity, unsigned long long* out_count)
{
  __shared__ unsigned long long base;
  const int64_t b = sb[blockIdx.y], e = se[blockIdx.y];
  for (int64_t c0 = b + (int64_t)blockIdx.x * kAppendChunk; c0 < e; c0 += (int64_t)gridDim.x * kAppendChunk) {
    const int n = (int)min((int64_t)kAppendChunk, e - c0);
    __syncthreads();  // `base` of the previous chunk has been read
    if (threadIdx.x == 0) base = atomicAdd(out_count, (unsigned long long)n);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t g = (int64_t)base + i;
      if (g < out_capacity) {
        const Row r = rows[c0 + i];
        out_key[g]  = r.key;
        out_pay[g]  = r.pay;
        if (out_sides) {
          null_key[g]  = 0;
          null_pay[g]  = 0;
          out_sides[g] = sides;
        }
      }
    }
  }
}

// After the last chunk of a streamed full outer join: every build (right) row whose bit in `bits` is
// clear was matched by no left row of any chunk, and is appended as (0, 0, key, payload) with sides
// kSideBuild.  The build side is walked bucket by bucket (the gaps between buckets hold stale rows);
// a block takes a bucket in tiles of kEmitTile rows, and reserves a tile's output rows with ONE
// global atomicAdd: the warps' ballots are scanned in shared memory.
constexpr int kEmitThreads = 256, kEmitPerThread = 4, kEmitTile = kEmitThreads * kEmitPerThread;

__global__ void __launch_bounds__(kEmitThreads) emit_unmatched_build_kernel(
  const Row* rows, const int64_t* bbeg, const int64_t* bend, int nbuckets, const uint32_t* bits, int64_t* null_key,
  int64_t* null_pay, int64_t* out_key, int64_t* out_pay, uint8_t* out_sides, int64_t out_capacity,
  unsigned long long* out_count)
{
  constexpr int kRuns = kEmitTile / 32;  // (warp, step) runs of 32 rows in a tile
  __shared__ unsigned long long run_base[kRuns];
  __shared__ int run_cnt[kRuns];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b = blockIdx.x; b < nbuckets; b += gridDim.x) {
    const int64_t b0 = bbeg[b], b1 = bend[b];
    for (int64_t t0 = b0; t0 < b1; t0 += kEmitTile) {
      int4 row[kEmitPerThread];
      unsigned lone[kEmitPerThread];
#pragma unroll
      for (int j = 0; j < kEmitPerThread; j++) {
        const int64_t r = t0 + j * kEmitThreads + threadIdx.x;
        bool mine       = false;
        row[j]          = make_int4(0, 0, 0, 0);
        if (r < b1 && !((bits[r >> 5] >> (r & 31)) & 1u)) {
          mine   = true;
          row[j] = __ldg(reinterpret_cast<const int4*>(rows + r));  // one 16-byte load per row
        }
        lone[j] = __ballot_sync(0xffffffffu, mine);
        if (lane == 0) run_cnt[j * (kEmitThreads / 32) + warp] = __popc(lone[j]);
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
      for (int j = 0; j < kEmitPerThread; j++) {
        if (!((lone[j] >> lane) & 1u)) continue;
        const int64_t g = (int64_t)run_base[j * (kEmitThreads / 32) + warp] + __popc(lone[j] & lanemask_lt());
        if (g < out_capacity) {
          null_key[g]  = 0;
          null_pay[g]  = 0;
          out_key[g]   = (int64_t)(((uint64_t)(uint32_t)row[j].y << 32) | (uint32_t)row[j].x);
          out_pay[g]   = (int64_t)(((uint64_t)(uint32_t)row[j].w << 32) | (uint32_t)row[j].z);
          out_sides[g] = kSideBuild;
        }
      }
      // the next tile writes run_base only past its first barrier, i.e. after every thread's reads above
    }
  }
}

}  // namespace

RadixPlan make_radix_plan(int64_t nbuild)
{
  const int target = join_shape() == 1 ? CfgB::kTargetRows : CfgA::kTargetRows;
  RadixPlan p{0, 0, 1};
  int bits = 0;
  while (bits < 20 && (nbuild >> bits) > target) bits++;
  if (bits <= 10) {
    p.bits1 = bits;
    p.bits2 = 0;
  } else {
    p.bits1 = bits / 2;
    p.bits2 = bits - p.bits1;
  }
  p.nbuckets = 1 << bits;
  return p;
}

int run_bucket_join(const JoinBuffers& jb, bool swap_output_sides, cudaStream_t stream)
{
  JoinDev d{};
  d.build    = jb.build;
  d.bbeg     = jb.d_build_begin;
  d.bend     = jb.d_build_end;
  d.probe    = jb.probe;
  d.pbeg     = jb.d_probe_begin;
  d.pend     = jb.d_probe_end;
  d.nbuckets = jb.nbuckets;
  for (int c = 0; c < 4; c++) d.out[c] = jb.out[swap_output_sides ? (c + 2) % 4 : c];
  d.out_capacity = jb.out_capacity;
  d.out_count    = (unsigned long long*)jb.d_out_count;
  d.probe_bits   = jb.d_probe_bits;
  d.out_sides    = jb.out_sides;
  d.build_bits   = jb.d_build_bits;
  return join_shape() == 1 ? launch_join_kind<CfgB>(d, jb.kind, 2, stream)
                           : launch_join_kind<CfgA>(d, jb.kind, 1, stream);
}

int append_segment_rows(const Row* rows, const int64_t* d_seg_begin, const int64_t* d_seg_end, int nseg,
                        int64_t max_seg_rows, int64_t* out_key, int64_t* out_pay, int64_t out_capacity,
                        int64_t* d_out_count, cudaStream_t stream, int64_t* null_key, int64_t* null_pay,
                        uint8_t* out_sides, uint8_t sides)
{
  if (nseg <= 0 || max_seg_rows <= 0) return DJ_OK;
  const int64_t chunks = (max_seg_rows + kAppendChunk - 1) / kAppendChunk;
  const dim3 grid((unsigned)(chunks < 64 ? chunks : 64), (unsigned)nseg);
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    append_rows_kernel<<<grid, 256, 0, stream>>>(rows, d_seg_begin, d_seg_end, out_key, out_pay, null_key, null_pay,
                                                 out_sides, sides, out_capacity, (unsigned long long*)d_out_count);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

int emit_unmatched_build(const Row* rows, const int64_t* d_begin, const int64_t* d_end, int nbuckets,
                         const uint32_t* d_build_bits, int64_t* const out[4], uint8_t* out_sides,
                         int64_t out_capacity, int64_t* d_out_count, cudaStream_t stream)
{
  if (nbuckets <= 0) return DJ_OK;
  const int grid = std::min(nbuckets, sm_count() * 8);
  {
    ProfScope prof(DJ_PROF_OTHER, stream);
    emit_unmatched_build_kernel<<<grid, kEmitThreads, 0, stream>>>(rows, d_begin, d_end, nbuckets, d_build_bits, out[0],
                                                                   out[1], out[2], out[3], out_sides, out_capacity,
                                                                   (unsigned long long*)d_out_count);
  }
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

const void* join_module_kernel() { return (const void*)bucket_join_kernel<CfgA, kInner>; }

}  // namespace dj
