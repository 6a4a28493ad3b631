// dj_internal.h -- host-side declarations shared between the .cu translation units.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/dj_b200.h"

namespace dj {

constexpr int kMaxPayload = 3;
constexpr int kMaxFanout  = 1024;

// Internal row format of everything between the caller's SoA columns and the join output:
// partitioned tables, exchanged pieces, radix levels and the join's inputs are arrays of 16-byte
// (key, payload) rows.  One row = one 128-bit access, a per-bucket run of rows is one contiguous
// 16-byte aligned range (a single cp.async.bulk in either direction), and an exchanged bucket is
// one copy instead of one per column.
struct __align__(16) Row {
  int64_t key;
  int64_t pay;
};

// Bucket function of one partition pass.
//   mode 0: (row_hash(key; seed, hash_id)) % F   -- the cuDF-compatible rank partition
//   mode 1: (local_hash(key) >> shift) & (F-1)   -- the join's private radix sub-partition
//   mode 2: ((row_hash % nparts) << sub_bits) | (local_hash >> (32 - sub_bits))
//           -- rank partition fused with the first local radix level (F = nparts << sub_bits)
struct PassDesc {
  int mode;
  uint32_t seed;
  int hash_id;
  int shift;
  int F;     // fan-out per parent bucket (<= kMaxFanout)
  int P;     // number of parent buckets (1 for a top-level pass, <= kMaxFanout)
  int npay;  // payload columns moved with the key (1..kMaxPayload)
  int align_rows = 1;  // child buckets start on multiples of this many rows (needs P*F <= 1024);
                       // in mode 2 only every destination's group of buckets is aligned
  int nparts   = 0;    // mode 2
  int sub_bits = 0;    // mode 2
};

struct PassBuffers {
  const int64_t* in_key;
  const int64_t* in_pay[kMaxPayload];
  int64_t* out_key;
  int64_t* out_pay[kMaxPayload];
  // Row-format (AoS) input / output; either replaces the SoA pointers of that side.  A pass with
  // out_rows set runs the row scatter kernel (key + one payload only).
  const Row* in_rows = nullptr;
  Row* out_rows      = nullptr;
  int64_t nrows;
  // [P] parent p is rows [d_parent_begin[p], d_parent_end[p]) of the input; nullptr when P == 1
  const int64_t* d_parent_begin = nullptr;
  const int64_t* d_parent_end   = nullptr;
  int64_t* d_child_off;         // [P*F+1] out: absolute row offsets of the child buckets
                                // (bounded passes: [P*F] first row of every child bucket)
  int64_t* d_child_end = nullptr;  // [P*F] out, bounded passes: one past every child bucket's last row
  // Optional explicit input segments (override the parent ranges): segment i is rows
  // [d_seg_begin[i], d_seg_end[i]) of the input and feeds output parent d_seg_parent[i]
  // (nullptr: parent 0).  Used for received tables, which are one padded piece per source rank.
  const int64_t* d_seg_begin = nullptr;
  const int64_t* d_seg_end   = nullptr;
  const int* d_seg_parent    = nullptr;
  int nseg                   = 0;
  int64_t* d_child_cnt       = nullptr;  // [P*F] out (aligned passes): rows per child bucket
};

// Device-side view of one pass (kernel argument).
struct PassDev {
  const int64_t* in_key;
  const int64_t* in_pay[kMaxPayload];
  int64_t* out_key;
  int64_t* out_pay[kMaxPayload];
  const Row* in_rows;        // row-format input (nullptr: SoA in_key / in_pay[0])
  Row* out_rows;             // row-format output (scatter_rows_kernel)
  // Fused partition + exchange: when set, bucket k's run goes to part_base[k >> part_shift] + cursor
  // instead of out_rows + cursor.  The bases are receive pieces -- local memory for this rank's own
  // part, CUDA-IPC mappings of the peers' workspaces for the others -- so the scatter kernel's
  // cp.async.bulk stores ARE the all-to-all: the TMA engine writes over NVLink.
  Row* const* part_base;
  int part_shift;
  int64_t in_total;          // rows in the input arrays (TMA windows are clamped to the column end)
  const int64_t* seg_begin;  // [S] first row of every input segment
  const int64_t* seg_end;    // [S] one past its last row
  const int* seg_parent;     // [S] output parent bucket the segment's rows belong to
  unsigned long long* counts;  // [P*F+1]
  unsigned long long* cursor;  // [P*F]
  // Bounded passes: a (tile, bucket) run whose reserved slice would pass cap_end[bucket] is not
  // copied; overflow[parent] is set instead (nullptr: exact offsets, no check).
  const unsigned long long* cap_end;
  int* overflow;
  const int* hist_tiles;       // [S+1] prefix of hist tiles per segment
  const int* scat_tiles;       // [S+1] prefix of scatter tiles per segment
  int S, P, F;
  uint32_t seed;
  int hash_id, shift, pow2;
  int nparts, sub_bits;  // mode 2: bucket = (row_hash % nparts) << sub_bits | top sub_bits of local_hash
};

// A pass runs in two stream-ordered halves so that callers can put work between them: the
// distributed join all-gathers the histogram's counts while the scatter kernels already run.
//   pass_histogram  tile plan + key histogram + child offsets (+ cursors)
//   pass_scatter    the scatter kernel
struct PassState {
  PassDev dev;
  int mode, npay;
  int64_t span;
};
int pass_histogram(const PassDesc& desc, const PassBuffers& buf, void* d_ws, size_t ws_bytes,
                   cudaStream_t stream, PassState* state);
int pass_scatter(const PassState& state, cudaStream_t stream);

size_t pass_workspace_bytes(int P, int F, int nseg = 0);
int run_partition_pass(const PassDesc& desc, const PassBuffers& buf, void* d_ws, size_t ws_bytes,
                       cudaStream_t stream);

// Bounded ("optimistic") radix pass, mode 1 with row output: no histogram.  Every child bucket gets
// a capacity from its parent's row count and the scatter runs at once; parents in which a child
// outgrew its capacity are re-scattered with exact offsets by stream-ordered repair kernels that
// return at once when nothing overflowed.  Child bucket i is rows [d_child_off[i], d_child_end[i]),
// with gaps between buckets.  `level` (0 or 1) only selects the repair counter.
int run_bounded_pass(const PassDesc& desc, const PassBuffers& buf, int level, void* d_ws, size_t ws_bytes,
                     cudaStream_t stream);
// Upper bound on the output rows of a bounded pass of `nrows` rows split into P parents x F children,
// whatever the parents' sizes.
int64_t bounded_pass_rows(int64_t nrows, int P, int F);
// Parents repaired per level since the previous read; reading clears the counts.
int read_radix_repairs(int64_t out[2]);

// Local join of radix-partitioned tables: bucket b of the build side is rows
// [d_build_begin[b], d_build_end[b]) of `build`, likewise for the probe side.
struct JoinBuffers {
  const Row* build;
  const int64_t* d_build_begin;
  const int64_t* d_build_end;
  const Row* probe;
  const int64_t* d_probe_begin;
  const int64_t* d_probe_end;
  int nbuckets;
  int64_t* out[4];  // build key, build payload, probe key, probe payload
  int64_t out_capacity;
  int64_t* d_out_count;    // running total (device); the kernel atomically adds to it
};
int run_bucket_join(const JoinBuffers& jb, bool swap_output_sides, cudaStream_t stream);

// Radix plan for a local join with `nbuild` build rows.
struct RadixPlan {
  int bits1, bits2;  // fan-out bits of level 1 / level 2 (0 = level not used)
  int nbuckets;
};
RadixPlan make_radix_plan(int64_t nbuild);

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// One side of a local join as it arrives: a contiguous table, or (received tables) `nseg` pieces
// [d_seg_begin[i], d_seg_end[i]) of arrays spanning `nrows` rows.
struct TableInput {
  const int64_t* key;  // SoA columns (the caller's table) ...
  const int64_t* pay;
  const Row* rows;     // ... or rows (a received table); exactly one of the two forms is set
  int64_t nrows;
  const int64_t* d_seg_begin;
  const int64_t* d_seg_end;
  int nseg;
  const int* d_seg_parent = nullptr;  // level-1 bucket of every segment (only with level1_done)
  bool level1_done        = false;    // the sender already split the rows into plan.bits1 buckets
};
// The same side radix-partitioned for the join: bucket b = rows [d_begin[b], d_end[b]).
struct PreparedSide {
  const Row* rows;
  const int64_t* d_begin;
  const int64_t* d_end;
};
RadixPlan plan_for(int64_t nbuild, bool any_segmented);
size_t side_ws_bytes(int64_t span_rows, const RadixPlan& plan, int nseg);

// Simple bump allocator over a caller-provided device workspace.
struct Arena {
  char* base;
  size_t size;
  size_t used = 0;
  Arena(void* p, size_t n) : base((char*)p), size(n) {}
  template <typename T>
  T* take(size_t count)
  {
    size_t off = align_up(used, 256);
    size_t end = off + count * sizeof(T);
    if (end > size) return nullptr;
    used = end;
    return (T*)(base + off);
  }
};


int prepare_side(const TableInput& in, const RadixPlan& plan, PreparedSide* out, Arena& arena,
                 cudaStream_t stream);
int join_prepared(const PreparedSide& build, const PreparedSide& probe, const RadixPlan& plan,
                  int64_t* const out[4], int64_t out_capacity, int64_t* d_out_count, bool swap,
                  cudaStream_t stream);
int local_join(const int64_t* bk, const int64_t* bp, int64_t nb, const int64_t* pk,
               const int64_t* pp, int64_t np, int64_t* const out[4], int64_t out_capacity,
               int64_t* d_out_count, bool swap, Arena& arena, cudaStream_t stream);
size_t local_join_workspace(int64_t nb, int64_t np);

// One kernel of each translation unit's module (partition.cu, join.cu, generate.cu): comm.cu
// loads every function of these modules before ranks can wait on each other.
const void* partition_module_kernel();
const void* join_module_kernel();
const void* generate_module_kernel();

}  // namespace dj
