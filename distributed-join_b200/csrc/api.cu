// api.cu -- C ABI entry points for the single-GPU stages (include/dj_b200.h):
// dj_hash_partition_i64 and dj_inner_join_i64, plus library bookkeeping.
#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "dj_device.cuh"
#include "dj_internal.h"

namespace dj {

static thread_local char g_error[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches += n; }

// ---- optional per-kernel event timing
static bool g_prof_on = false;
struct ProfRec { int cat; cudaEvent_t a, b; };
static std::vector<ProfRec> g_prof_recs;
static std::vector<cudaEvent_t> g_prof_pool;
static std::mutex g_prof_mu;

static cudaEvent_t prof_event()
{
  if (!g_prof_pool.empty()) {
    cudaEvent_t e = g_prof_pool.back();
    g_prof_pool.pop_back();
    return e;
  }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}

ProfScope::ProfScope(int category, cudaStream_t st) : cat(category), stream(st), slot(-1)
{
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfRec r{cat, prof_event(), prof_event()};
  cudaEventRecord(r.a, stream);
  g_prof_recs.push_back(r);
  slot = (int)g_prof_recs.size() - 1;
}

ProfScope::~ProfScope()
{
  if (slot < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEventRecord(g_prof_recs[slot].b, stream);
}

// SMs deliberately left idle by the persistent partition kernels while an NCCL exchange is in
// flight, so that NCCL's copy kernels can become resident next to them (see comm.cu).
static thread_local int g_sm_reserve = 0;
void set_sm_reserve(int n) { g_sm_reserve = n < 0 ? 0 : n; }

int sm_count()
{
  const int total = sm_count_physical();
  const int keep  = total - g_sm_reserve;
  return keep < total / 2 ? total / 2 : keep;
}

int sm_count_physical()
{
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;  // H100 SXM
  if (dev != cached_dev) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 132;
    cached     = prop.multiProcessorCount;
    cached_dev = dev;
  }
  return cached;
}


// Radix plan shared by both sides of one local join.  Every side goes through at least one pass:
// it is the pass that turns the caller's SoA columns (or the padded per-source pieces of a
// received table) into the contiguous row-format buckets the join kernel streams.
//
// A semi / anti / outer join builds on the right table, which is often tiny next to the left one (a fact
// table filtered by a small key set).  The join kernel runs at most one CTA per bucket, so its
// plan gets at least kFilterMinBits bits (1024 buckets: every SM busy with either CTA shape); a
// bucket then holds less than one build job, and the probe side is spread over all of them.
RadixPlan join_plan(int kind, int64_t nbuild)
{
  RadixPlan plan = make_radix_plan(nbuild);
  if (plan.bits1 == 0) {
    plan.bits1    = 1;
    plan.nbuckets = 2;
  }
  if (kind && plan.bits1 + plan.bits2 < kFilterMinBits) {
    plan.bits1    = kFilterMinBits;
    plan.bits2    = 0;
    plan.nbuckets = 1 << kFilterMinBits;
  }
  return plan;
}

// rows of the array prepare_side lays a side of `span_rows` rows out into (bucket gaps included)
static int64_t prepared_rows(int64_t span_rows, const RadixPlan& plan)
{
  const int F1 = 1 << plan.bits1, F2 = 1 << plan.bits2;
  return (plan.bits2 ? bounded_pass_rows(span_rows, F1, F2) : bounded_pass_rows(span_rows, 1, F1)) + 8;
}

size_t filter_bits_bytes(int64_t span_rows, const RadixPlan& plan)
{
  return align_up((size_t)((prepared_rows(span_rows, plan) + 31) / 32) * 4, 256) + 256;
}

// DJ_RADIX_EXACT=1: the join's radix levels size their buckets with exact histograms instead of
// capacities (for A/B comparison and tests)
static bool radix_exact()
{
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DJ_RADIX_EXACT");
    v             = (e && e[0] == '1') ? 1 : 0;
  }
  return v == 1;
}

// scratch for one side: partition passes' outputs (capacity-padded: bounded_pass_rows), bucket
// ranges and pass workspaces
size_t side_ws_bytes(int64_t span_rows, const RadixPlan& plan, int nseg)
{
  const int F1 = 1 << plan.bits1, F2 = 1 << plan.bits2;
  size_t total = 4096;
  total += align_up((size_t)(bounded_pass_rows(span_rows, 1, F1) + 8) * sizeof(Row), 256);
  if (plan.bits2) total += align_up((size_t)(bounded_pass_rows(span_rows, F1, F2) + 8) * sizeof(Row), 256);
  total += 2 * align_up(((size_t)plan.nbuckets + 1) * 8, 256) + 2 * align_up(((size_t)F1 + 1) * 8, 256);
  size_t pw = pass_workspace_bytes(1, F1, nseg);
  if (plan.bits2) pw = std::max(pw, pass_workspace_bytes(F1, F2, nseg));
  return total + pw + 1024;
}

size_t local_join_workspace(int kind, int64_t nbuild, int64_t nprobe)
{
  const RadixPlan plan = join_plan(kind, nbuild);
  return side_ws_bytes(nbuild, plan, 0) + side_ws_bytes(nprobe, plan, 0) +
         (kind ? filter_bits_bytes(nprobe, plan) : 0) + 8192;
}

// Radix-partitions one side of a join into plan.nbuckets row-format buckets (1 or 2 passes).  By
// default every pass is bounded (run_bounded_pass: no histogram, buckets with gaps); with
// DJ_RADIX_EXACT=1 every pass is exact and bucket b ends where bucket b+1 begins.
int prepare_side(const TableInput& in, const RadixPlan& plan, PreparedSide* out, Arena& arena,
                 cudaStream_t stream)
{
  const int F1 = 1 << plan.bits1, F2 = 1 << plan.bits2;
  DJ_REQUIRE(plan.bits1 > 0, "inner_join: a radix plan needs at least one level");
  DJ_REQUIRE(!in.level1_done || (plan.bits2 && in.d_seg_parent && in.rows),
             "inner_join: fused level 1 needs a two-level plan and row-format pieces");
  const bool exact = radix_exact();
  const bool two   = plan.bits2 > 0 && !in.level1_done;  // this side runs both levels
  auto ranges = [&](size_t n, int64_t** end) {  // bucket begins; ends are the next begins when exact
    int64_t* b = arena.take<int64_t>(n + 1);
    *end       = exact ? (b ? b + 1 : nullptr) : arena.take<int64_t>(n);
    return b;
  };
  int64_t *end = nullptr, *end1 = nullptr;
  int64_t* beg  = ranges((size_t)plan.nbuckets, &end);
  int64_t* beg1 = two ? ranges((size_t)F1, &end1) : nullptr;
  const size_t pw = std::max(pass_workspace_bytes(1, F1, in.nseg),
                             plan.bits2 ? pass_workspace_bytes(F1, F2, in.nseg) : (size_t)0);
  char* pass_ws = arena.take<char>(pw);
  Row* r1 = two ? arena.take<Row>((size_t)bounded_pass_rows(in.nrows, 1, F1) + 8) : nullptr;
  const int64_t rows_out = prepared_rows(in.nrows, plan);
  Row* r = arena.take<Row>((size_t)rows_out);
  if (!beg || !end || (two && (!beg1 || !end1 || !r1)) || !pass_ws || !r) {
    set_error("inner_join: workspace too small");
    return DJ_ERR_WORKSPACE;
  }
  // one radix pass of P parents x F children into `dst`; bucket i = [cb[i], ce[i])
  auto pass = [&](PassBuffers pb, int level, int P, int F, int shift, Row* dst, int64_t* cb, int64_t* ce) {
    PassDesc d{1, 0, 0, shift, F, P, 1};
    pb.out_rows    = dst;
    pb.d_child_off = cb;
    if (exact) return run_partition_pass(d, pb, pass_ws, pw, stream);
    pb.d_child_end = ce;
    return run_bounded_pass(d, pb, level, pass_ws, pw, stream);
  };
  PassBuffers pb{};
  pb.in_rows   = in.rows;
  pb.in_key    = in.key;
  pb.in_pay[0] = in.pay;
  pb.nrows     = in.nrows;
  if (in.nseg > 0) {
    pb.d_seg_begin  = in.d_seg_begin;
    pb.d_seg_end    = in.d_seg_end;
    pb.d_seg_parent = in.d_seg_parent;
    pb.nseg         = in.nseg;
  }
  out->rows     = r;
  out->d_begin  = beg;
  out->d_end    = end;
  out->cap_rows = rows_out;
  // the exchange delivered level-1 buckets as (source, bucket) segments: run level 2 only
  if (in.level1_done) return pass(pb, 1, F1, F2, 32 - plan.bits1 - plan.bits2, r, beg, end);
  pb.d_seg_parent = nullptr;  // a first level has a single parent
  if (!two) return pass(pb, 0, 1, F1, 32 - plan.bits1, r, beg, end);
  int rc = pass(pb, 0, 1, F1, 32 - plan.bits1, r1, beg1, end1);
  if (rc) return rc;
  PassBuffers pb2{};
  pb2.in_rows        = r1;
  pb2.nrows          = bounded_pass_rows(in.nrows, 1, F1);
  pb2.d_parent_begin = beg1;
  pb2.d_parent_end   = end1;
  return pass(pb2, 1, F1, F2, 32 - plan.bits1 - plan.bits2, r, beg, end);
}

int join_prepared(int kind, const PreparedSide& build, const PreparedSide& probe, const RadixPlan& plan,
                  int64_t* const out[4], uint8_t* out_sides, int64_t out_capacity, int64_t* d_out_count, bool swap,
                  Arena& arena, cudaStream_t stream, uint32_t* d_build_bits)
{
  const bool filter = kind_is_filter(kind), outer = kind && !filter;  // outer: kJoinFullOuterMark included
  JoinBuffers jb{};
  jb.build = build.rows; jb.d_build_begin = build.d_begin; jb.d_build_end = build.d_end;
  jb.probe = probe.rows; jb.d_probe_begin = probe.d_begin; jb.d_probe_end = probe.d_end;
  jb.nbuckets = plan.nbuckets;
  for (int c = 0; c < 4; c++) jb.out[c] = filter && c >= 2 ? nullptr : out[c];
  jb.out_capacity = out_capacity;
  jb.d_out_count  = d_out_count;
  jb.kind         = kind;
  jb.out_sides    = outer ? out_sides : nullptr;
  jb.d_build_bits = d_build_bits;
  if (kind) {  // one zeroed bit per prepared probe row
    const size_t words = (size_t)(probe.cap_rows + 31) / 32;
    jb.d_probe_bits    = arena.take<uint32_t>(words);
    if (!jb.d_probe_bits) {
      set_error("join: workspace too small for the probe-row bits");
      return DJ_ERR_WORKSPACE;
    }
    DJ_CUDA_TRY(cudaMemsetAsync(jb.d_probe_bits, 0, words * 4, stream));
  }
  // the kernel writes (build row, probe row): an outer join's build side is the right table, so its
  // output is swapped into left ++ right; a semi / anti join writes probe rows only
  return run_bucket_join(jb, kind ? outer : swap, stream);
}

int local_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* rk, const int64_t* rp,
               int64_t nr, int64_t* const out[4], uint8_t* out_sides, int64_t out_capacity, int64_t* d_out_count,
               bool build_right, Arena& arena, cudaStream_t stream)
{
  const bool right = build_right || kind;
  const TableInput tl{lk, lp, nullptr, nl, nullptr, nullptr, 0}, tr{rk, rp, nullptr, nr, nullptr, nullptr, 0};
  const TableInput& tb = right ? tr : tl;
  const TableInput& tp = right ? tl : tr;
  const RadixPlan plan = join_plan(kind, tb.nrows);
  PreparedSide sb{}, sp{};
  int rc = prepare_side(tb, plan, &sb, arena, stream);
  if (rc) return rc;
  rc = prepare_side(tp, plan, &sp, arena, stream);
  if (rc) return rc;
  return join_prepared(kind, sb, sp, plan, out, out_sides, out_capacity, d_out_count, right, arena, stream);
}

}  // namespace dj

using namespace dj;

extern "C" int dj_version(void) { return DJ_VERSION; }
extern "C" const char* dj_last_error(void) { return dj::g_error; }
extern "C" int64_t dj_kernel_launch_count(void) { return dj::g_launches.load(); }

extern "C" int dj_profile_enable(int on)
{
  std::lock_guard<std::mutex> lk(dj::g_prof_mu);
  dj::g_prof_on = on != 0;
  return DJ_OK;
}

extern "C" int dj_profile_read(double* h_ms4, int64_t* h_launches4)
{
  std::lock_guard<std::mutex> lk(dj::g_prof_mu);
  for (int c = 0; c < DJ_PROF_NCAT; c++) {
    h_ms4[c]       = 0;
    h_launches4[c] = 0;
  }
  for (auto& r : dj::g_prof_recs) {
    DJ_CUDA_TRY(cudaEventSynchronize(r.b));
    float ms = 0;
    DJ_CUDA_TRY(cudaEventElapsedTime(&ms, r.a, r.b));
    h_ms4[r.cat] += ms;
    h_launches4[r.cat] += 1;
    dj::g_prof_pool.push_back(r.a);
    dj::g_prof_pool.push_back(r.b);
  }
  dj::g_prof_recs.clear();
  return DJ_OK;
}

extern "C" int dj_testing_radix_repairs(int64_t* h_out2)
{
  DJ_REQUIRE(h_out2, "radix_repairs: bad argument");
  return read_radix_repairs(h_out2);
}

extern "C" size_t dj_hash_partition_workspace_bytes(int64_t nrows, int nparts)
{
  (void)nrows;
  if (nparts < 1) nparts = 1;
  return pass_workspace_bytes(1, nparts) + 4096;
}

extern "C" int dj_hash_partition_i64(const int64_t* d_key, const int64_t* const* h_payload_cols,
                                     int npayload, int64_t nrows, int nparts, uint32_t seed,
                                     int hash_id, int64_t* d_out_key,
                                     int64_t* const* h_out_payload_cols, int64_t* d_offsets,
                                     void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(nparts >= 1 && nparts <= kMaxFanout, "hash_partition: nparts %d not in [1, %d]", nparts,
             kMaxFanout);
  DJ_REQUIRE(npayload >= 1 && npayload <= kMaxPayload,
             "hash_partition: %d payload columns (supported: 1..%d)", npayload, kMaxPayload);
  DJ_REQUIRE(hash_id == DJ_HASH_MURMUR3 || hash_id == DJ_HASH_IDENTITY, "hash_partition: bad hash id");
  DJ_REQUIRE(nrows >= 0 && d_offsets && d_workspace, "hash_partition: bad argument");
  PassDesc desc{0, seed, hash_id, 0, nparts, 1, npayload};
  PassBuffers buf{};
  buf.in_key  = d_key;
  buf.out_key = d_out_key;
  for (int c = 0; c < npayload; c++) {
    buf.in_pay[c]  = h_payload_cols[c];
    buf.out_pay[c] = h_out_payload_cols[c];
  }
  buf.nrows       = nrows;
  buf.d_child_off = d_offsets;
  return run_partition_pass(desc, buf, d_workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" size_t dj_inner_join_workspace_bytes(int64_t nbuild, int64_t nprobe)
{
  return local_join_workspace(0, nbuild, nprobe);
}

extern "C" int dj_inner_join_i64(const int64_t* d_build_key, const int64_t* d_build_payload,
                                 int64_t nbuild, const int64_t* d_probe_key,
                                 const int64_t* d_probe_payload, int64_t nprobe,
                                 int64_t* d_out_build_key, int64_t* d_out_build_payload,
                                 int64_t* d_out_probe_key, int64_t* d_out_probe_payload,
                                 int64_t out_capacity, int64_t* d_out_count, void* d_workspace,
                                 size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(nbuild >= 0 && nprobe >= 0 && out_capacity >= 0 && d_out_count, "inner_join: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  DJ_CUDA_TRY(cudaMemsetAsync(d_out_count, 0, sizeof(int64_t), st));
  if (nbuild == 0 || nprobe == 0) return DJ_OK;  // src/distributed_join.cpp:76-82
  DJ_REQUIRE(d_workspace, "inner_join: workspace missing");
  Arena arena(d_workspace, workspace_bytes);
  int64_t* out[4] = {d_out_build_key, d_out_build_payload, d_out_probe_key, d_out_probe_payload};
  return local_join(0, d_build_key, d_build_payload, nbuild, d_probe_key, d_probe_payload, nprobe, out, nullptr,
                    out_capacity, d_out_count, false, arena, st);
}
