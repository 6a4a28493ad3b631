// api.cu -- C ABI entry points for the single-GPU stages (include/dj_b200.h):
// dj_hash_partition_i64 and dj_inner_join_i64, plus library bookkeeping.
#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>
#include <cstdarg>
#include <cstdio>

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
RadixPlan plan_for(int64_t nbuild, bool /*any_segmented*/)
{
  RadixPlan plan = make_radix_plan(nbuild);
  if (plan.bits1 == 0) {
    plan.bits1    = 1;
    plan.nbuckets = 2;
  }
  return plan;
}

// scratch for one side: partition passes' outputs, offsets and pass workspaces
size_t side_ws_bytes(int64_t span_rows, const RadixPlan& plan, int nseg)
{
  const int levels = (plan.bits1 > 0) + (plan.bits2 > 0);
  const int F1 = 1 << plan.bits1, F2 = 1 << plan.bits2;
  size_t total = 4096;
  total += (size_t)levels * align_up((size_t)span_rows * sizeof(Row) + 256, 256);
  total += align_up(((size_t)plan.nbuckets + 1) * 8, 256) + align_up(((size_t)F1 + 1) * 8, 256);
  size_t pw = pass_workspace_bytes(1, F1, nseg);
  if (plan.bits2) pw = std::max(pw, pass_workspace_bytes(F1, F2, nseg));
  return total + pw + 1024;
}

static size_t local_join_ws_bytes(int64_t nb, int64_t np)
{
  const RadixPlan plan = plan_for(nb, false);
  return side_ws_bytes(nb, plan, 0) + side_ws_bytes(np, plan, 0) + 8192;
}

// Radix-partitions one side of a join into plan.nbuckets row-format buckets (1 or 2 passes).
int prepare_side(const TableInput& in, const RadixPlan& plan, PreparedSide* out, Arena& arena,
                 cudaStream_t stream)
{
  const int F1 = 1 << plan.bits1, F2 = 1 << plan.bits2;
  DJ_REQUIRE(plan.bits1 > 0, "inner_join: a radix plan needs at least one level");
  int64_t* off = arena.take<int64_t>((size_t)plan.nbuckets + 1);
  const size_t pw = std::max(pass_workspace_bytes(1, F1, in.nseg),
                             plan.bits2 ? pass_workspace_bytes(F1, F2, in.nseg) : (size_t)0);
  char* pass_ws = arena.take<char>(pw);
  if (!off || !pass_ws) {
    set_error("inner_join: workspace too small");
    return DJ_ERR_WORKSPACE;
  }
  out->d_off = off;
  auto set_input = [&](PassBuffers& pb) {
    pb.in_rows = in.rows;
    pb.in_key  = in.key;
    pb.in_pay[0] = in.pay;
    pb.nrows   = in.nrows;
    if (in.nseg > 0) {
      pb.d_seg_begin  = in.d_seg_begin;
      pb.d_seg_end    = in.d_seg_end;
      pb.d_seg_parent = in.d_seg_parent;
      pb.nseg         = in.nseg;
    }
  };
  if (in.level1_done) {
    // the exchange delivered level-1 buckets as (source, bucket) segments: run level 2 only
    if (!plan.bits2 || !in.d_seg_parent || !in.rows) {
      set_error("inner_join: fused level 1 needs a two-level plan and row-format pieces");
      return DJ_ERR_ARG;
    }
    Row* r2 = arena.take<Row>((size_t)in.nrows + 8);
    if (!r2) {
      set_error("inner_join: workspace too small");
      return DJ_ERR_WORKSPACE;
    }
    PassDesc d2{1, 0, 0, 32 - plan.bits1 - plan.bits2, F2, F1, 1};
    PassBuffers pb2{};
    set_input(pb2);
    pb2.out_rows = r2;
    pb2.d_child_off = off;
    int rc2 = run_partition_pass(d2, pb2, pass_ws, pw, stream);
    if (rc2) return rc2;
    out->rows = r2;
    return DJ_OK;
  }
  Row* r1       = arena.take<Row>((size_t)in.nrows + 8);
  int64_t* off1 = plan.bits2 ? arena.take<int64_t>((size_t)F1 + 1) : off;
  if (!r1 || !off1) {
    set_error("inner_join: workspace too small");
    return DJ_ERR_WORKSPACE;
  }
  PassDesc d1{1, 0, 0, 32 - plan.bits1, F1, 1, 1};
  PassBuffers pb{};
  set_input(pb);
  pb.d_seg_parent = nullptr;  // a first level has a single parent
  pb.out_rows     = r1;
  pb.d_child_off  = off1;
  int rc = run_partition_pass(d1, pb, pass_ws, pw, stream);
  if (rc) return rc;
  out->rows = r1;
  if (plan.bits2) {
    Row* r2 = arena.take<Row>((size_t)in.nrows + 8);
    if (!r2) {
      set_error("inner_join: workspace too small");
      return DJ_ERR_WORKSPACE;
    }
    PassDesc d2{1, 0, 0, 32 - plan.bits1 - plan.bits2, F2, F1, 1};
    PassBuffers pb2{};
    pb2.in_rows = r1; pb2.out_rows = r2;
    pb2.nrows = in.nrows; pb2.d_parent_off = off1; pb2.d_child_off = off;
    rc = run_partition_pass(d2, pb2, pass_ws, pw, stream);
    if (rc) return rc;
    out->rows = r2;
  }
  return DJ_OK;
}

int join_prepared(const PreparedSide& build, const PreparedSide& probe, const RadixPlan& plan,
                  int64_t* const out[4], int64_t out_capacity, int64_t* d_out_count, bool swap,
                  cudaStream_t stream)
{
  JoinBuffers jb{};
  jb.build = build.rows; jb.d_build_off = build.d_off;
  jb.probe = probe.rows; jb.d_probe_off = probe.d_off;
  jb.nbuckets = plan.nbuckets;
  for (int c = 0; c < 4; c++) jb.out[c] = out[c];
  jb.out_capacity = out_capacity;
  jb.d_out_count  = d_out_count;
  return run_bucket_join(jb, swap, stream);
}

// Joins (bk,bp)[nb] with (pk,pp)[np]; appends matches at *d_out_count (running, device).
// out[] is always (left key, left payload, right key, right payload); when swap is true the
// build side is the caller's RIGHT table.
int local_join(const int64_t* bk, const int64_t* bp, int64_t nb, const int64_t* pk,
               const int64_t* pp, int64_t np, int64_t* const out[4], int64_t out_capacity,
               int64_t* d_out_count, bool swap, Arena& arena, cudaStream_t stream)
{
  if (nb == 0 || np == 0) return DJ_OK;  // src/distributed_join.cpp:76-82
  const RadixPlan plan = plan_for(nb, false);
  TableInput tb{bk, bp, nullptr, nb, nullptr, nullptr, 0}, tp{pk, pp, nullptr, np, nullptr, nullptr, 0};
  PreparedSide sb{}, sp{};
  int rc = prepare_side(tb, plan, &sb, arena, stream);
  if (rc) return rc;
  rc = prepare_side(tp, plan, &sp, arena, stream);
  if (rc) return rc;
  return join_prepared(sb, sp, plan, out, out_capacity, d_out_count, swap, stream);
}

size_t local_join_workspace(int64_t nb, int64_t np) { return local_join_ws_bytes(nb, np); }

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
  buf.nrows        = nrows;
  buf.d_parent_off = nullptr;
  buf.d_child_off  = d_offsets;
  return run_partition_pass(desc, buf, d_workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" size_t dj_inner_join_workspace_bytes(int64_t nbuild, int64_t nprobe)
{
  return local_join_ws_bytes(nbuild, nprobe);
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
  if (nbuild == 0 || nprobe == 0) return DJ_OK;
  DJ_REQUIRE(d_workspace, "inner_join: workspace missing");
  Arena arena(d_workspace, workspace_bytes);
  int64_t* out[4] = {d_out_build_key, d_out_build_payload, d_out_probe_key, d_out_probe_payload};
  return local_join(d_build_key, d_build_payload, nbuild, d_probe_key, d_probe_payload, nprobe, out,
                    out_capacity, d_out_count, false, arena, st);
}
