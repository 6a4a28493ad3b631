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
  // 0: inner join.  DJ_JOIN_LEFT_SEMI / DJ_JOIN_LEFT_ANTI: the build side is the right table, out[0..1]
  // receive the probe (left) rows, and d_probe_bits holds one zeroed bit per row of `probe`.
  // DJ_JOIN_LEFT_OUTER / DJ_JOIN_FULL_OUTER: the build side is the right table, d_probe_bits as for
  // semi / anti, and out_sides receives every output row's DJ_SIDE_* bits.
  int kind               = 0;
  uint32_t* d_probe_bits = nullptr;
  uint8_t* out_sides     = nullptr;
  // kJoinFullOuterMark: one bit per row POSITION of `build` (gaps between buckets included); the
  // kernel sets the bits of the build rows it matched and never clears one
  uint32_t* d_build_bits = nullptr;
};
// A join kind of the library's own, not of the ABI: one left chunk of a full outer join whose left
// table arrives in several launches.  Its output is a left outer join's; the right rows it matched
// are recorded in JoinBuffers::d_build_bits, and emit_unmatched_build appends the right rows no
// launch matched once the last chunk has been joined.
constexpr int kJoinFullOuterMark = DJ_JOIN_FULL_OUTER + 1;
int run_bucket_join(const JoinBuffers& jb, bool swap_output_sides, cudaStream_t stream);
// Appends the rows of segments [d_seg_begin[i], d_seg_end[i]) (each at most max_seg_rows long) to
// (out_key, out_pay) at the running count *d_out_count, in no particular order.  With out_sides set
// (outer joins), the same output rows of (null_key, null_pay) are zeroed and their sides byte is set.
int append_segment_rows(const Row* rows, const int64_t* d_seg_begin, const int64_t* d_seg_end, int nseg,
                        int64_t max_seg_rows, int64_t* out_key, int64_t* out_pay, int64_t out_capacity,
                        int64_t* d_out_count, cudaStream_t stream, int64_t* null_key = nullptr,
                        int64_t* null_pay = nullptr, uint8_t* out_sides = nullptr, uint8_t sides = 0);

// Appends every row of buckets [d_begin[b], d_end[b]) of `rows` whose bit in d_build_bits (indexed by
// row position) is clear as (0, 0, key, payload) with sides DJ_SIDE_RIGHT, at the running count.
int emit_unmatched_build(const Row* rows, const int64_t* d_begin, const int64_t* d_end, int nbuckets,
                         const uint32_t* d_build_bits, int64_t* const out[4], uint8_t* out_sides,
                         int64_t out_capacity, int64_t* d_out_count, cudaStream_t stream);

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
  int64_t cap_rows;  // length of the `rows` array (bucket gaps included)
};
// The radix plan of a local join of `kind` with `nbuild` build rows.  Semi / anti / outer joins get
// at least kFilterMinBits bits, so that the probe side is spread over every SM however small the
// right table is.
constexpr int kFilterMinBits = 10;
RadixPlan join_plan(int kind, int64_t nbuild);
size_t side_ws_bytes(int64_t span_rows, const RadixPlan& plan, int nseg);
// bytes of the probe-row bit array of a semi / anti / outer join for a probe side spanning `span_rows` rows
size_t filter_bits_bytes(int64_t span_rows, const RadixPlan& plan);

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
// The join kernel of `kind` over two prepared sides; appends at the running *d_out_count.  out is
// (left key, left payload, right key, right payload); semi / anti joins write only out[0..1].  Every
// kind but the inner join builds on the right table; the inner join does when `swap` is set.  Kinds
// other than the inner join take their probe-row bit array from `arena` and zero it; outer joins
// write every row's DJ_SIDE_* bits to out_sides, and kJoinFullOuterMark also takes d_build_bits,
// (build.cap_rows + 31) / 32 words zeroed once by the caller.
int join_prepared(int kind, const PreparedSide& build, const PreparedSide& probe, const RadixPlan& plan,
                  int64_t* const out[4], uint8_t* out_sides, int64_t out_capacity, int64_t* d_out_count, bool swap,
                  Arena& arena, cudaStream_t stream, uint32_t* d_build_bits = nullptr);
// Single-GPU join of `kind` of (lk, lp)[nl] with (rk, rp)[nr], both non-empty; semi / anti joins pass
// the right key column as rp.  The inner join builds on the right table when `build_right` is set,
// every other kind always does.  Its workspace is local_join_workspace(kind, nbuild, nprobe).
int local_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* rk, const int64_t* rp,
               int64_t nr, int64_t* const out[4], uint8_t* out_sides, int64_t out_capacity, int64_t* d_out_count,
               bool build_right, Arena& arena, cudaStream_t stream);
size_t local_join_workspace(int kind, int64_t nbuild, int64_t nprobe);

// Which side the hash tables of an inner join are built on.  The caller's LEFT table is the build side
// (the reference's drivers pass the unique-key build table as `left`, benchmark/distributed_join.cu:266-283)
// unless the right table is clearly smaller: received slices of equal-sized tables differ by a few rows
// per rank, and letting that noise pick the side made some ranks build on the duplicate-laden probe
// table (measured at N=2: 11.2 ms instead of 7.9 ms for the same join).
inline bool build_on_right(int64_t nleft, int64_t nright) { return nright + nright / 8 < nleft; }

// The ABI's join kinds: 0 (inner), DJ_JOIN_LEFT_SEMI / ANTI (two output columns, the right table is a
// key column) and DJ_JOIN_LEFT_OUTER / FULL_OUTER (four columns and the sides bytes).
inline bool kind_is_filter(int kind) { return kind == DJ_JOIN_LEFT_SEMI || kind == DJ_JOIN_LEFT_ANTI; }
inline bool kind_is_outer(int kind) { return kind == DJ_JOIN_LEFT_OUTER || kind == DJ_JOIN_FULL_OUTER; }
inline int kind_out_cols(int kind) { return kind_is_filter(kind) ? 2 : 4; }

// The distributed join of every kind (comm.cu).  kind 0: out = (left key, left payload, right key,
// right payload).  Semi / anti: d_right_payload == d_right_key, out[0..1] receive the kept left rows.
// Outer: out as for the inner join, d_out_sides receives every row's DJ_SIDE_* bits.
int distributed_join(dj_comm_t* comm, int kind, const int64_t* d_left_key, const int64_t* d_left_payload,
                     int64_t nleft, const int64_t* d_right_key, const int64_t* d_right_payload, int64_t nright,
                     int64_t* d_out_lk, int64_t* d_out_lp, int64_t* d_out_rk, int64_t* d_out_rp, uint8_t* d_out_sides,
                     int64_t out_capacity, int64_t* h_out_count, dj_join_options* opts, void* d_workspace,
                     size_t workspace_bytes, void* stream);
// Zeroes every output field of a join's options (nullptr: none).
void reset_opts(dj_join_options* opts);
// A single-rank join's result of n rows: *h_out_count = n, DJ_ERR_OVERFLOW (with the error set) if it
// exceeds out_capacity.
int single_rank_result(int64_t n, int64_t out_capacity, int64_t* h_out_count);

// Broadcast join's local join (broadcast.cu): a hash table of the distinct keys of the right table
// (rk, rp)[nr], nr <= DJ_BROADCAST_TABLE_MAX_ROWS, probed by the left columns (lk, lp)[nl] in place.
// kind 0 / DJ_JOIN_LEFT_SEMI / DJ_JOIN_LEFT_ANTI / DJ_JOIN_LEFT_OUTER; out and out_sides as for the
// repartitioned join of that kind (rp, out[2..3] and out_sides unused by semi / anti); appends at the
// running *d_out_count.  Takes broadcast_table_bytes(nr) from `arena`.
size_t broadcast_table_bytes(int64_t nr);
int broadcast_hash_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* rk,
                        const int64_t* rp, int64_t nr, int64_t* const out[4], uint8_t* out_sides,
                        int64_t out_capacity, int64_t* d_out_count, Arena& arena, cudaStream_t stream);

// One kernel of each translation unit's module (partition.cu, join.cu, generate.cu, broadcast.cu):
// comm.cu loads every function of these modules before ranks can wait on each other.
const void* partition_module_kernel();
const void* join_module_kernel();
const void* generate_module_kernel();
const void* broadcast_module_kernel();

}  // namespace dj
