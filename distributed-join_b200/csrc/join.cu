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
#include <cstdlib>

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
};

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

template <int N>
__device__ __forceinline__ void consumer_sync()
{
  asm volatile("bar.sync 1, %0;" ::"n"(N) : "memory");
}

// Build jobs of the cached descriptor block: (bucket, build chunk) pairs whose bucket is
// non-empty on both sides.  Every thread walks them identically.
template <class S>
__device__ __forceinline__ int next_valid_bucket(const S& s, int lb, int nd)
{
  while (lb < nd && (s.dbe[lb] == s.dbb[lb] || s.dpe[lb] == s.dpb[lb])) lb++;
  return lb;
}

// Slot word: bit 31 = occupied, bits 30..11 = 20-bit key fingerprint, bits 10..0 = build row.
__device__ __forceinline__ uint32_t slot_tag(uint32_t h) { return 0x100000u | (h >> 12); }

template <class C>
__global__ void __launch_bounds__(C::kThreads, 1) bucket_join_kernel(JoinDev d)
{
  using Smem = JoinSmem<C>;
  constexpr int kConsumers = C::kConsumers;
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
        for (int lb = next_valid_bucket(s, 0, nd); lb < nd; lb = next_valid_bucket(s, lb + 1, nd)) {
          const int64_t b1 = s.dbe[lb], p0 = s.dpb[lb], p1 = s.dpe[lb];
          for (int64_t c0 = s.dbb[lb]; c0 < b1; c0 += C::kBuildChunk) {
            {
              const int bs = u & 1;
              const int n  = (int)min((int64_t)C::kBuildChunk, b1 - c0);
              mbar_wait(&s.empty_build[bs], ((u >> 1) & 1) ^ 1);
              mbar_expect_tx(&s.full_build[bs], (uint32_t)n * 16u);
              tma_load(s.brow[bs], d.build + c0, (uint32_t)n * 16u, &s.full_build[bs]);
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
      for (int lb = next_valid_bucket(s, 0, nd); lb < nd; lb = next_valid_bucket(s, lb + 1, nd)) {
        const int64_t b1 = s.dbe[lb], p0 = s.dpb[lb], p1 = s.dpe[lb];
        for (int64_t c0 = s.dbb[lb]; c0 < b1; c0 += C::kBuildChunk) {
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
          if (lane == 0) mbar_arrive(&s.empty_build[bs]);
          if (pend_n) {
            // copy out the tile whose atomicAdd was issued one build job ago (latency hidden);
            // it stays untouched until the job after next, when every thread is past here
            const int64_t gb = (int64_t)s.sbase[pend_tile];
#pragma unroll
            for (int c = 0; c < 4; c++)
              for (int i = tid; i < pend_n; i += kConsumers)
                if (gb + i < d.out_capacity) d.out[c][gb + i] = s.sout[pend_tile][c][i];
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
      for (int c = 0; c < 4; c++)
        for (int i = tid; i < pend_n; i += kConsumers)
          if (gb + i < d.out_capacity) d.out[c][gb + i] = s.sout[pend_tile][c][i];
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

template <class C>
int launch_join(const JoinDev& d, int ctas_per_sm, cudaStream_t stream)
{
  const size_t smem = sizeof(JoinSmem<C>);
  auto kern         = bucket_join_kernel<C>;
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
  return join_shape() == 1 ? launch_join<CfgB>(d, 2, stream) : launch_join<CfgA>(d, 1, stream);
}

const void* join_module_kernel() { return (const void*)bucket_join_kernel<CfgA>; }

}  // namespace dj
