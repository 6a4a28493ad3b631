// host_join.cu -- the distributed join entries that take and return HOST columns
// (include/dj_b200.h): one rank streams the tables through the GPU, more ranks stage them in front of
// the device join's workspace.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "dj_device.cuh"
#include "dj_internal.h"

using namespace dj;

static size_t streamed_ws_bytes(int kind, int64_t nleft, int64_t nright, int64_t out_capacity);

// bytes host_join_staged puts in front of the device join's workspace (same arithmetic as its arena walk)
static size_t staged_prefix_bytes(int kind, int64_t nleft, int64_t nright, int64_t out_capacity)
{
  return 2 * align_up((size_t)nleft * 8, 256) + (kind_is_filter(kind) ? 1 : 2) * align_up((size_t)nright * 8, 256) +
         kind_out_cols(kind) * align_up((size_t)out_capacity * 8, 256) +
         (kind_is_outer(kind) ? align_up((size_t)out_capacity, 256) : 0);
}

extern "C" size_t dj_distributed_inner_join_host_workspace_bytes(int64_t nleft, int64_t nright,
                                                                 int64_t out_capacity, int world,
                                                                 int over_decom_factor)
{
  const size_t staged = dj_distributed_inner_join_workspace_bytes(nleft, nright, world, over_decom_factor) +
                        staged_prefix_bytes(0, nleft, nright, out_capacity) + 8192;
  if (world > 1) return staged;
  return std::max(staged, streamed_ws_bytes(0, nleft, nright, out_capacity));
}

// One rank streams and stages nothing; more ranks stage the columns in front of the device join's workspace.
extern "C" size_t dj_distributed_left_filter_join_host_workspace_bytes(int64_t nleft, int64_t nright,
                                                                       int64_t out_capacity, int world,
                                                                       int over_decom_factor)
{
  if (world <= 1) return streamed_ws_bytes(DJ_JOIN_LEFT_SEMI, nleft, nright, out_capacity);
  return dj_distributed_left_filter_join_workspace_bytes(nleft, nright, world, over_decom_factor) +
         staged_prefix_bytes(DJ_JOIN_LEFT_SEMI, nleft, nright, out_capacity);
}

// Sized for a full outer join, which needs the build-row bits on top of what a left outer join needs.
extern "C" size_t dj_distributed_outer_join_host_workspace_bytes(int64_t nleft, int64_t nright,
                                                                 int64_t out_capacity, int world,
                                                                 int over_decom_factor)
{
  if (world <= 1) return streamed_ws_bytes(DJ_JOIN_FULL_OUTER, nleft, nright, out_capacity);
  return dj_distributed_outer_join_workspace_bytes(nleft, nright, world, over_decom_factor) +
         staged_prefix_bytes(DJ_JOIN_FULL_OUTER, nleft, nright, out_capacity);
}

// Single-GPU end-to-end join with HOST tables, streamed: the PCIe link is the bottleneck (25.6 GB in,
// 7.7 GB out at 800M x 800M against ~50 ms of GPU work), so the call is organised around keeping
// both directions of the link busy:
//   1. the build table goes up first and is radix-partitioned while the probe table's first chunks
//      are already on the wire;
//   2. the probe table goes up in chunks (double-buffered); each chunk is partitioned with the same
//      radix plan and joined against the resident build buckets as soon as it has landed -- the GPU
//      re-inserts the build rows once per chunk, which costs HBM bandwidth that is idle anyway;
//   3. each chunk's matches go down on their own stream while the next chunk comes up (full duplex).
// What is left after the last byte has arrived is one chunk's join and one chunk's matches.
//
// Every kind but the inner join builds on the right table and chunks the left one.  For semi, anti
// and left outer joins a left row's fate depends on the whole right table only, so a chunk's rows
// are final when its join ends.  A full outer join's right rows are the exception: a right row is
// unmatched only if no chunk matched it.  Its chunks run as kJoinFullOuterMark, which records the
// matched build rows in one bit array for the whole call, and after the last chunk
// emit_unmatched_build appends the rows whose bit is clear; they go down as one more drain.
struct StreamedShape {
  bool swap;
  int64_t nb, np, chunk;
  int nchunks;
  RadixPlan plan;
};
static StreamedShape streamed_shape(int kind, int64_t nleft, int64_t nright)
{
  StreamedShape s{};
  s.swap      = kind ? true : build_on_right(nleft, nright);
  s.nb        = s.swap ? nright : nleft;
  s.np        = s.swap ? nleft : nright;
  s.plan      = join_plan(kind, s.nb > 0 ? s.nb : 1);
  int nchunks = 16;
  const char* e = getenv("DJ_HOST_CHUNKS");
  if (e && atoi(e) > 0) nchunks = atoi(e);
  int64_t chunk = (s.np + nchunks - 1) / nchunks;
  if (chunk < (1 << 20)) chunk = std::min<int64_t>(s.np, 1 << 20);  // small tables: few chunks
  chunk     = std::max<int64_t>((chunk + 1) / 2 * 2, 2);  // even row counts keep the host columns 16-byte aligned
  s.chunk   = chunk;
  s.nchunks = (int)std::max<int64_t>((s.np + chunk - 1) / chunk, 1);
  return s;
}
// device bytes host_join_streamed takes from the workspace (same arithmetic as its arena walk)
static size_t streamed_ws_bytes(int kind, int64_t nleft, int64_t nright, int64_t out_capacity)
{
  const StreamedShape s = streamed_shape(kind, nleft, nright);
  size_t total = 256 + (kind_is_filter(kind) ? 1 : 2) * align_up((size_t)s.nb * 8, 256);
  total += (s.nchunks > 1 ? 4 : 2) * align_up((size_t)s.chunk * 8, 256);
  total += kind_out_cols(kind) * align_up((size_t)out_capacity * 8, 256);
  if (kind_is_outer(kind)) total += align_up((size_t)out_capacity, 256);
  total += side_ws_bytes(s.nb, s.plan, 0) + side_ws_bytes(s.chunk, s.plan, 0);
  if (kind == DJ_JOIN_FULL_OUTER) total += filter_bits_bytes(s.nb, s.plan);  // build-row bits, whole call
  if (kind) total += filter_bits_bytes(s.chunk, s.plan);                     // probe-row bits, one chunk
  return total + (64 << 10);
}

// A semi, anti or outer join with an empty table: the result is the other table's rows (anti and
// outer joins keep every left row of an empty right table, a full outer join every right row of an
// empty left table) or nothing.  Host columns to host columns, no kernel.
static int host_join_empty_side(int kind, const int64_t* h_left_key, const int64_t* h_left_payload, int64_t nleft,
                                const int64_t* h_right_key, const int64_t* h_right_payload, int64_t nright,
                                int64_t* const h_out[4], uint8_t* h_out_sides, int64_t out_capacity,
                                int64_t* h_out_count, cudaStream_t st)
{
  const bool left_rows  = nright == 0 && kind != DJ_JOIN_LEFT_SEMI;
  const bool right_rows = nleft == 0 && kind == DJ_JOIN_FULL_OUTER;
  const int64_t total   = left_rows ? nleft : right_rows ? nright : 0;
  const size_t n        = (size_t)std::min(total, out_capacity);
  DJ_CUDA_TRY(cudaStreamSynchronize(st));  // the caller's stream orders the call
  if (n > 0) {
    const int at = left_rows ? 0 : 2;  // columns of the present side
    memcpy(h_out[at], left_rows ? h_left_key : h_right_key, n * 8);
    memcpy(h_out[at + 1], left_rows ? h_left_payload : h_right_payload, n * 8);
    if (kind_is_outer(kind)) {
      memset(h_out[2 - at], 0, n * 8);
      memset(h_out[3 - at], 0, n * 8);
      memset(h_out_sides, left_rows ? DJ_SIDE_LEFT : DJ_SIDE_RIGHT, n);
    }
  }
  return single_rank_result(total, out_capacity, h_out_count);
}

static int host_join_streamed(int kind, const int64_t* h_left_key, const int64_t* h_left_payload, int64_t nleft,
                              const int64_t* h_right_key, const int64_t* h_right_payload, int64_t nright,
                              int64_t* const h_out[4], uint8_t* h_out_sides, int64_t out_capacity,
                              int64_t* h_out_count, dj_join_options* opts, void* d_workspace, size_t workspace_bytes,
                              cudaStream_t st)
{
  *h_out_count = 0;
  reset_opts(opts);
  if (kind && (nleft == 0 || nright == 0))
    return host_join_empty_side(kind, h_left_key, h_left_payload, nleft, h_right_key, h_right_payload, nright, h_out,
                                h_out_sides, out_capacity, h_out_count, st);
  if (nleft == 0 || nright == 0) return DJ_OK;  // src/distributed_join.cpp:76-82
  const StreamedShape shape = streamed_shape(kind, nleft, nright);
  const bool swap      = shape.swap;
  const int64_t nb     = shape.nb, np = shape.np, chunk = shape.chunk;
  const int nchunks    = shape.nchunks;
  const bool filter    = kind_is_filter(kind), outer = kind_is_outer(kind), full = kind == DJ_JOIN_FULL_OUTER;
  const int ncols      = kind_out_cols(kind);
  const int nsteps     = nchunks + (full ? 1 : 0);  // joins, and the full outer join's unmatched right rows
  const int64_t* h_bk  = swap ? h_right_key : h_left_key;
  const int64_t* h_bp  = swap ? h_right_payload : h_left_payload;
  const int64_t* h_pk  = swap ? h_left_key : h_right_key;
  const int64_t* h_pp  = swap ? h_left_payload : h_right_payload;
  const RadixPlan plan = shape.plan;
  const size_t ws_need = streamed_ws_bytes(kind, nleft, nright, out_capacity);
  auto ws_too_small = [&]() {
    set_error("distributed join (host): workspace too small (%zu bytes given, %zu needed)", workspace_bytes, ws_need);
    if (opts) opts->workspace_needed = (int64_t)ws_need;
    return DJ_ERR_WORKSPACE;
  };
  // the semi / anti / outer entries take exactly what their query returns; the inner entry, as ever,
  // whatever its arena walk fits into
  if (kind && workspace_bytes < ws_need) return ws_too_small();
  int64_t* h_cnt = nullptr;  // pinned: running match count after every step (allocated before any work is queued)
  DJ_CUDA_TRY(cudaMallocHost(&h_cnt, (size_t)(nsteps + 1) * 8));
  struct PinGuard {
    int64_t* p;
    ~PinGuard() { cudaFreeHost(p); }
  } pin_guard{h_cnt};

  Arena arena(d_workspace, workspace_bytes);
  int64_t* d_count = arena.take<int64_t>(32);
  int64_t* dbk     = arena.take<int64_t>((size_t)nb);
  int64_t* dbp     = filter ? dbk : arena.take<int64_t>((size_t)nb);  // a key column is its own payload
  int64_t* dck[2], *dcp[2];
  for (int i = 0; i < 2; i++) {  // one buffer is enough for a single chunk
    dck[i] = (i == 0 || nchunks > 1) ? arena.take<int64_t>((size_t)chunk) : dck[0];
    dcp[i] = (i == 0 || nchunks > 1) ? arena.take<int64_t>((size_t)chunk) : dcp[0];
  }
  int64_t* o[4] = {nullptr, nullptr, nullptr, nullptr};
  bool taken = d_count && dbk && dbp && dck[0] && dcp[0] && dck[1] && dcp[1];
  for (int c = 0; c < ncols; c++) taken = (o[c] = arena.take<int64_t>((size_t)out_capacity)) && taken;
  uint8_t* o_sides = outer ? arena.take<uint8_t>((size_t)out_capacity) : nullptr;
  if (!taken || (outer && !o_sides)) return ws_too_small();
  cudaStream_t up = nullptr, down = nullptr;
  std::vector<cudaEvent_t> ev;  // [0] build up, then per step: landed, partitioned, joined
  auto cleanup = [&]() {
    for (auto e : ev) cudaEventDestroy(e);
    if (up) cudaStreamDestroy(up);
    if (down) cudaStreamDestroy(down);
  };
  struct Guard {
    decltype(cleanup)& f;
    ~Guard() { f(); }
  } guard{cleanup};
  DJ_CUDA_TRY(cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking));
  DJ_CUDA_TRY(cudaStreamCreateWithFlags(&down, cudaStreamNonBlocking));
  ev.resize(2 + (size_t)nsteps * 3, nullptr);
  for (auto& e : ev) DJ_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  cudaEvent_t ev_start = ev[1];
  auto ev_landed = [&](int c) { return ev[2 + (size_t)c * 3]; };
  auto ev_parted = [&](int c) { return ev[3 + (size_t)c * 3]; };
  auto ev_joined = [&](int c) { return ev[4 + (size_t)c * 3]; };

  // the caller's stream orders the call: uploads start after whatever it had queued
  DJ_CUDA_TRY(cudaEventRecord(ev_start, st));
  DJ_CUDA_TRY(cudaStreamWaitEvent(up, ev_start, 0));
  DJ_CUDA_TRY(cudaStreamWaitEvent(down, ev_start, 0));
  DJ_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), st));
  DJ_CUDA_TRY(cudaMemcpyAsync(dbk, h_bk, (size_t)nb * 8, cudaMemcpyHostToDevice, up));
  if (!filter) DJ_CUDA_TRY(cudaMemcpyAsync(dbp, h_bp, (size_t)nb * 8, cudaMemcpyHostToDevice, up));
  DJ_CUDA_TRY(cudaEventRecord(ev[0], up));

  // build side: partitioned once, resident for the whole call
  PreparedSide build{}, probe{};
  DJ_CUDA_TRY(cudaStreamWaitEvent(st, ev[0], 0));
  TableInput tb{dbk, dbp, nullptr, nb, nullptr, nullptr, 0};
  int rc = prepare_side(tb, plan, &build, arena, st);
  if (rc) return rc;
  uint32_t* build_bits = nullptr;  // full outer: the build rows some chunk matched, zeroed once per call
  if (full) {
    const size_t words = (size_t)(build.cap_rows + 31) / 32;
    build_bits         = arena.take<uint32_t>(words);
    if (!build_bits) return ws_too_small();
    DJ_CUDA_TRY(cudaMemsetAsync(build_bits, 0, words * 4, st));
  }
  const size_t chunk_mark = arena.used;
  int64_t done_rows = 0;  // output rows already on their way to the host
  auto drain = [&](int c) -> int {  // step c's rows -> host, on the download stream
    DJ_CUDA_TRY(cudaEventSynchronize(ev_joined(c)));
    int64_t upto = h_cnt[c] < out_capacity ? h_cnt[c] : out_capacity;
    if (upto > done_rows) {
      DJ_CUDA_TRY(cudaStreamWaitEvent(down, ev_joined(c), 0));
      for (int col = 0; col < ncols; col++)
        DJ_CUDA_TRY(cudaMemcpyAsync(h_out[col] + done_rows, o[col] + done_rows, (size_t)(upto - done_rows) * 8,
                                    cudaMemcpyDeviceToHost, down));
      if (outer)
        DJ_CUDA_TRY(cudaMemcpyAsync(h_out_sides + done_rows, o_sides + done_rows, (size_t)(upto - done_rows),
                                    cudaMemcpyDeviceToHost, down));
      done_rows = upto;
    }
    return DJ_OK;
  };
  for (int c = 0; c < nchunks; c++) {
    const int64_t r0 = (int64_t)c * chunk, n = std::min(chunk, np - r0);
    const int bi     = c & 1;
    if (c >= 2) DJ_CUDA_TRY(cudaStreamWaitEvent(up, ev_parted(c - 2), 0));  // the buffer's previous chunk is consumed
    DJ_CUDA_TRY(cudaMemcpyAsync(dck[bi], h_pk + r0, (size_t)n * 8, cudaMemcpyHostToDevice, up));
    DJ_CUDA_TRY(cudaMemcpyAsync(dcp[bi], h_pp + r0, (size_t)n * 8, cudaMemcpyHostToDevice, up));
    DJ_CUDA_TRY(cudaEventRecord(ev_landed(c), up));

    DJ_CUDA_TRY(cudaStreamWaitEvent(st, ev_landed(c), 0));
    arena.used = chunk_mark;  // probe scratch (and the probe-row bits) are reused chunk after chunk (same stream)
    TableInput tp{dck[bi], dcp[bi], nullptr, n, nullptr, nullptr, 0};
    rc = prepare_side(tp, plan, &probe, arena, st);
    if (rc) return rc;
    DJ_CUDA_TRY(cudaEventRecord(ev_parted(c), st));
    rc = join_prepared(full ? kJoinFullOuterMark : kind, build, probe, plan, o, o_sides, out_capacity, d_count, swap,
                       arena, st, build_bits);
    if (rc) return rc;
    DJ_CUDA_TRY(cudaMemcpyAsync(h_cnt + c, d_count, 8, cudaMemcpyDeviceToHost, st));
    DJ_CUDA_TRY(cudaEventRecord(ev_joined(c), st));
    // the previous chunk's matches go down while this chunk is being joined and the next comes up
    if (c >= 1 && (rc = drain(c - 1))) return rc;
  }
  if (full) {
    // every chunk has set its bits: the right rows nobody matched, while the last chunk's rows go down
    rc = emit_unmatched_build(build.rows, build.d_begin, build.d_end, plan.nbuckets, build_bits, o, o_sides,
                              out_capacity, d_count, st);
    if (rc) return rc;
    DJ_CUDA_TRY(cudaMemcpyAsync(h_cnt + nchunks, d_count, 8, cudaMemcpyDeviceToHost, st));
    DJ_CUDA_TRY(cudaEventRecord(ev_joined(nchunks), st));
    if ((rc = drain(nchunks - 1))) return rc;
  }
  if ((rc = drain(nsteps - 1))) return rc;
  DJ_CUDA_TRY(cudaStreamSynchronize(down));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  return single_rank_result(h_cnt[nsteps - 1], out_capacity, h_out_count);
}

// N > 1: stage the columns at the front of the workspace, run the device entry of `kind` on the rest,
// copy min(count, capacity) rows down (also under DJ_ERR_OVERFLOW).
static int host_join_staged(dj_comm_t* comm, int kind, const int64_t* h_left_key, const int64_t* h_left_payload,
                            int64_t nleft, const int64_t* h_right_key, const int64_t* h_right_payload, int64_t nright,
                            int64_t* const h_out[4], uint8_t* h_out_sides, int64_t out_capacity, int64_t* h_out_count,
                            dj_join_options* opts, void* d_workspace, size_t workspace_bytes, cudaStream_t st)
{
  const bool filter = kind_is_filter(kind), outer = kind_is_outer(kind);
  const int ncols   = kind_out_cols(kind);
  Arena arena(d_workspace, workspace_bytes);
  int64_t* dlk = arena.take<int64_t>((size_t)nleft);
  int64_t* dlp = arena.take<int64_t>((size_t)nleft);
  int64_t* drk = arena.take<int64_t>((size_t)nright);
  int64_t* drp = filter ? drk : arena.take<int64_t>((size_t)nright);
  int64_t* o[4] = {nullptr, nullptr, nullptr, nullptr};
  bool taken = dlk && dlp && drk && drp;
  for (int c = 0; c < ncols; c++) taken = (o[c] = arena.take<int64_t>((size_t)out_capacity)) && taken;
  uint8_t* o_sides = outer ? arena.take<uint8_t>((size_t)out_capacity) : nullptr;
  if (!taken || (outer && !o_sides)) {
    // unlike the join's own verdict this one is local: size the workspace with the entry's
    // *_host_workspace_bytes, which always leaves room for the staging
    set_error("distributed join (host): workspace too small for the staged columns");
    return DJ_ERR_WORKSPACE;
  }
  DJ_CUDA_TRY(cudaMemcpyAsync(dlk, h_left_key, (size_t)nleft * 8, cudaMemcpyHostToDevice, st));
  DJ_CUDA_TRY(cudaMemcpyAsync(dlp, h_left_payload, (size_t)nleft * 8, cudaMemcpyHostToDevice, st));
  DJ_CUDA_TRY(cudaMemcpyAsync(drk, h_right_key, (size_t)nright * 8, cudaMemcpyHostToDevice, st));
  if (!filter) DJ_CUDA_TRY(cudaMemcpyAsync(drp, h_right_payload, (size_t)nright * 8, cudaMemcpyHostToDevice, st));
  const size_t off = align_up(arena.used, 256);
  int rc = distributed_join(comm, kind, dlk, dlp, nleft, drk, drp, nright, o[0], o[1], o[2], o[3], o_sides,
                            out_capacity, h_out_count, opts, (char*)d_workspace + off, workspace_bytes - off, st);
  // the device join sized only what follows the staged columns: report the whole workspace
  if (rc == DJ_ERR_WORKSPACE && opts && opts->workspace_needed > 0) opts->workspace_needed += (int64_t)off;
  if (rc && rc != DJ_ERR_OVERFLOW) return rc;
  const int64_t n = *h_out_count < out_capacity ? *h_out_count : out_capacity;
  for (int c = 0; c < ncols; c++)
    DJ_CUDA_TRY(cudaMemcpyAsync(h_out[c], o[c], (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  if (outer) DJ_CUDA_TRY(cudaMemcpyAsync(h_out_sides, o_sides, (size_t)n, cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  return rc;
}

// One rank streams; more ranks stage in, join on the device, stage out.
static int host_join(dj_comm_t* comm, int kind, const int64_t* h_left_key, const int64_t* h_left_payload,
                     int64_t nleft, const int64_t* h_right_key, const int64_t* h_right_payload, int64_t nright,
                     int64_t* const h_out[4], uint8_t* h_out_sides, int64_t out_capacity, int64_t* h_out_count,
                     dj_join_options* opts, void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(d_workspace && h_out_count && nleft >= 0 && nright >= 0, "distributed join (host): bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (dj_comm_size(comm) == 1)
    return host_join_streamed(kind, h_left_key, h_left_payload, nleft, h_right_key, h_right_payload, nright, h_out,
                              h_out_sides, out_capacity, h_out_count, opts, d_workspace, workspace_bytes, st);
  return host_join_staged(comm, kind, h_left_key, h_left_payload, nleft, h_right_key, h_right_payload, nright, h_out,
                          h_out_sides, out_capacity, h_out_count, opts, d_workspace, workspace_bytes, st);
}

extern "C" int dj_distributed_inner_join_i64_host(
  dj_comm_t* comm, const int64_t* h_left_key, const int64_t* h_left_payload, int64_t nleft,
  const int64_t* h_right_key, const int64_t* h_right_payload, int64_t nright, int64_t* h_out_lk,
  int64_t* h_out_lp, int64_t* h_out_rk, int64_t* h_out_rp, int64_t out_capacity,
  int64_t* h_out_count, dj_join_options* opts, void* d_workspace, size_t workspace_bytes,
  void* stream)
{
  int64_t* h[4] = {h_out_lk, h_out_lp, h_out_rk, h_out_rp};
  return host_join(comm, 0, h_left_key, h_left_payload, nleft, h_right_key, h_right_payload, nright, h, nullptr,
                   out_capacity, h_out_count, opts, d_workspace, workspace_bytes, stream);
}

extern "C" int dj_distributed_left_filter_join_i64_host(dj_comm_t* comm, int kind, const int64_t* h_left_key,
                                                        const int64_t* h_left_payload, int64_t nleft,
                                                        const int64_t* h_right_key, int64_t nright,
                                                        int64_t* h_out_key, int64_t* h_out_payload,
                                                        int64_t out_capacity, int64_t* h_out_count,
                                                        dj_join_options* opts, void* d_workspace,
                                                        size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(kind_is_filter(kind), "left_filter_join_host: unknown join kind %d", kind);
  DJ_REQUIRE(out_capacity >= 0 && (out_capacity == 0 || (h_out_key && h_out_payload)),
             "left_filter_join_host: bad output columns");
  int64_t* h[4] = {h_out_key, h_out_payload, nullptr, nullptr};
  return host_join(comm, kind, h_left_key, h_left_payload, nleft, h_right_key, h_right_key, nright, h, nullptr,
                   out_capacity, h_out_count, opts, d_workspace, workspace_bytes, stream);
}

extern "C" int dj_distributed_outer_join_i64_host(dj_comm_t* comm, int kind, const int64_t* h_left_key,
                                                  const int64_t* h_left_payload, int64_t nleft,
                                                  const int64_t* h_right_key, const int64_t* h_right_payload,
                                                  int64_t nright, int64_t* h_out_lk, int64_t* h_out_lp,
                                                  int64_t* h_out_rk, int64_t* h_out_rp, uint8_t* h_out_sides,
                                                  int64_t out_capacity, int64_t* h_out_count, dj_join_options* opts,
                                                  void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(kind_is_outer(kind), "outer_join_host: unknown join kind %d", kind);
  DJ_REQUIRE(out_capacity >= 0 &&
               (out_capacity == 0 || (h_out_lk && h_out_lp && h_out_rk && h_out_rp && h_out_sides)),
             "outer_join_host: bad output columns");
  int64_t* h[4] = {h_out_lk, h_out_lp, h_out_rk, h_out_rp};
  return host_join(comm, kind, h_left_key, h_left_payload, nleft, h_right_key, h_right_payload, nright, h,
                   h_out_sides, out_capacity, h_out_count, opts, d_workspace, workspace_bytes, stream);
}
